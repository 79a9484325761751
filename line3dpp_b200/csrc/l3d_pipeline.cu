// l3d_pipeline.cu — the per-view scoring sweep of Line3D::computeMatches (line3D.cc:702-778) on the device.
//
// After l3d_match_pairs has produced the kNN match records of every view pair in one launch, the reference walks the
// views in ascending camID order and, for each view: filters its matches by orientation (checkMatchOrientation,
// line3D.cc:811-858), sorts them by (tgt cam, tgt seg) and flattens them (scoringGPU, 1311-1355), scores them
// (K_score_matches, cudawrapper.cu:256-367), hands the positively scored ones to the not-yet-processed target views as
// inverse matches (storeInverseMatches, 1672-1699) and keeps the good ones + the best 3D estimate per segment
// (filterMatches, 1586-1669).
//
// What really depends on the view order is ONE bit per inverse match: "did its source score it > 0".  Everything else is
// hoisted out of the chain and done for ALL views at once:
//   k_sw_flags      orientation check of every record from both sides; sizes of the (view, segment, neighbour) chunks
//   cub scan        chunk offsets = the final list layout of every view (l3d_sweep.cuh)
//   k_sw_scatter    records -> their chunk(s);  k_sw_chunksort: the (<= kNN-ish) entries of a chunk into list order
//   ---- chain: ONE launch per view, in camID order --------------------------------------------------------------
//   k_sw_score      a warp per segment stages the segment's list in shared memory (3D direction, target regulariser,
//                   depths: what scoringGPU's host pass + K_score_matches' prologue compute), scores every active entry
//                   against it with K_score_matches' loop, publishes score3D, the view's maximum and - the only thing the
//                   next views need - the "active" bit of the inverse entries it creates
//   ---- after the chain, all views at once -----------------------------------------------------------------------
//   k_sw_filter     filterMatches + the best 3D estimate per segment
//
// Arithmetic contract as in l3d_device.cuh (-fmad=false): the float parts repeat K_score_matches operation by
// operation (same libdevice expf/acosf), the double parts repeat the host code of view.cc / line3D.cc (IEEE double, no
// contraction); pinned against the unmodified reference in tests/test_ref_full_gpu.py.
#include "l3d_cub.cuh"
#include "l3d_device_f64.cuh"
#include "l3d_sweep.cuh"

#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>

#define L3D_PI_1_32_F 0.098174771f
#define L3D_PI_31_32_F 3.043417886f

// per-segment double rays, computed once per sweep: View::getNormalizedRay (view.cc:317-321) of the two end points and of the
// mid point (segmentQualityAngle, view.cc:466-484) - the same values the orientation check and View::unprojectSegment
// (view.cc:356-371) would recompute per match
struct SegRaysQ { D3 r1, r2, rm; };
__global__ void __launch_bounds__(256)
k_sw_rays(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, int V, long long N, double* __restrict__ rays, float4* __restrict__ rmf)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    const L3DViewDev* Vw = views + last_le(V, g, [&](int i) { return views[i].seg_off; });
    const float4 s = segs[g];
    const D3 r1 = dray(Vw->RtKinv_d, (double)s.x, (double)s.y), r2 = dray(Vw->RtKinv_d, (double)s.z, (double)s.w);
    const D3 rm = dray(Vw->RtKinv_d, 0.5 * ((double)s.x + (double)s.z), 0.5 * ((double)s.y + (double)s.w));
    double* o = rays + 9 * g;
    o[0] = r1.x; o[1] = r1.y; o[2] = r1.z; o[3] = r2.x; o[4] = r2.y; o[5] = r2.z; o[6] = rm.x; o[7] = rm.y; o[8] = rm.z;
    rmf[g] = make_float4((float)rm.x, (float)rm.y, (float)rm.z, 0.f);
}
__device__ __forceinline__ SegRaysQ sw_load_rays(const double* __restrict__ rays, long long g)
{
    const double* p = rays + 9 * g;
    SegRaysQ q;
    q.r1 = d3(__ldg(p), __ldg(p + 1), __ldg(p + 2)); q.r2 = d3(__ldg(p + 3), __ldg(p + 4), __ldg(p + 5)); q.rm = d3(__ldg(p + 6), __ldg(p + 7), __ldg(p + 8));
    return q;
}
// the end points View::unprojectSegment (view.cc:356-371) computes, with the cached rays; seg3d() makes the Segment3D of them
__device__ __forceinline__ void sw_unproject_pts(const L3DViewDev* v, const SegRaysQ& q, float d1, float d2, D3* P1, D3* P2)
{
    const D3 C = d3(v->C_d[0], v->C_d[1], v->C_d[2]);
    *P1 = d3(C.x + q.r1.x * (double)d1, C.y + q.r1.y * (double)d1, C.z + q.r1.z * (double)d1);
    *P2 = d3(C.x + q.r2.x * (double)d2, C.y + q.r2.y * (double)d2, C.z + q.r2.z * (double)d2);
}

// checkMatchOrientation (line3D.cc:811-858) for the match (segment of view V with rays q, depths d1,d2): unprojectMatch
// (1556-1568) + View::segmentQualityAngle (view.cc:466-484): keep iff pi/32 < acos(clamp(ray_mid . dir)) < 31 pi/32.
// acos is monotonic: away from the two thresholds the decision follows from the cosine alone (margin 1e-9 >> the few ulps by
// which the shortcut's cosine, one division instead of three, can differ from the reference's); inside the margins the
// reference's own sequence decides.
__device__ __forceinline__ bool sw_orientation_ok(const L3DViewDev* V, const SegRaysQ& q, float d1, float d2)
{
    D3 P1, P2;
    sw_unproject_pts(V, q, d1, d2, &P1, &P2);
    const D3 d = dsub(P2, P1);
    const double n2 = ddot(d, d);
    if (n2 > 1e-20) {
        const double c = ddot(q.rm, d) / sqrt(n2);
        // the cosines of the thresholds the reference compares acos with, (double)L3D_PI_1_32_F and (double)L3D_PI_31_32_F: the two
        // float constants are not symmetric about pi/2, so c2 != -c1
        const double c1 = 0.99518472640441780, c2 = -0.99518473132192450;
        if (c < c1 - 1e-9 && c > c2 + 1e-9) return true;
        if (c > c1 + 1e-9 || c < c2 - 1e-9) return false;
    }
    const double ang = acos(fmin(fmax(ddot(q.rm, seg3d(P1, P2).dir), -1.0), 1.0));
    return ang > (double)L3D_PI_1_32_F && ang < (double)L3D_PI_31_32_F;
}

// ---------------------------------------------------------------------------------------------- batched set-up kernels
// What the record-parallel set-up kernels need to know about a pair.  The table (one entry per pair) and the first pair of every
// thread block are built on the HOST once per sweep: with them a thread reaches its pair without walking
// pairs[p] -> views[src] -> vt[src] ... as a chain of dependent global loads and without any block-level synchronisation.
struct SwPairInfo {
    long long row_off, row_end, src_seg_off, tgt_seg_off, src_chunk_base, tgt_chunk_base;
    int src, tgt, src_np, tgt_np, cx, cy;
};
#define SW_SETUP_THREADS 256
__device__ __forceinline__ SwPairInfo sw_pair_info(const SwPairInfo* __restrict__ pinfo, const int* __restrict__ block_pair0, long long row)
{
    int p = __ldg(block_pair0 + blockIdx.x);
    while (row >= pinfo[p].row_end) ++p;            // a block of consecutive record slots touches one pair, rarely two
    return pinfo[p];
}

// Orientation check decided in FLOAT where that is safe: the angle between the mid-point ray and the 3D direction does not
// depend on the camera centre (d = r2*d2 - r1*d1), the float rays differ from the double ones by ~1e-7, and for |d| > 1 % of the
// depths the cosine is good to ~1e-5 - two orders below the 1e-4 margin kept around cos(pi/32).  Returns 1 keep, 0 drop, -1 undecided.
__device__ __forceinline__ int sw_orientation_fast(float3 r1, float3 r2, float3 rm, float d1, float d2)
{
    const float3 d = make_float3(r2.x * d2 - r1.x * d1, r2.y * d2 - r1.y * d1, r2.z * d2 - r1.z * d1);
    const float n2 = d.x * d.x + d.y * d.y + d.z * d.z;
    if (!(n2 > 1e-4f * (d1 * d1 + d2 * d2))) return -1;
    const float c = fabsf((rm.x * d.x + rm.y * d.y + rm.z * d.z) * rsqrtf(n2));
    if (c < 0.99518473f - 1e-4f) return 1;
    if (c > 0.99518473f + 1e-4f) return 0;
    return -1;
}

// P1: one thread per record slot.  rflag bit 0: the record survives the orientation check as a direct match of its source
// view, bit 1: as an inverse match of its target view (only asked for when the target is processed after the source).
__global__ void __launch_bounds__(256)
k_sw_flags(const double* __restrict__ rays, const float4* __restrict__ cache, const float4* __restrict__ rmf, const L3DViewDev* __restrict__ views,
           const SwPairInfo* __restrict__ pinfo, const int* __restrict__ block_pair0, const int* __restrict__ counts, const l3d_match_rec* __restrict__ recs,
           int knn, long long slots, unsigned char* __restrict__ rflag, int* __restrict__ csize)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= slots) return;
    const long long row = g / knn;
    const int i = (int)(g - row * knn);
    if (i >= counts[row]) return;
    const l3d_match_rec rec = recs[g];
    const SwPairInfo q = sw_pair_info(pinfo, block_pair0, row);
    const int r = (int)(row - q.row_off);
    unsigned char f = 0;
    {
        const long long gs = q.src_seg_off + r;
        const SegRays R = load_rays(cache, gs);
        const float4 m = __ldg(rmf + gs);
        int ok = sw_orientation_fast(R.r1, R.r2, make_float3(m.x, m.y, m.z), rec.d_p1, rec.d_p2);
        if (ok < 0) ok = sw_orientation_ok(views + q.src, sw_load_rays(rays, gs), rec.d_p1, rec.d_p2) ? 1 : 0;
        if (ok) { f |= 1; atomicAdd(csize + q.src_chunk_base + (long long)r * q.src_np + q.cx, 1); }
    }
    if (q.cy >= 0) {
        const long long gs = q.tgt_seg_off + rec.tgt_seg;
        const SegRays R = load_rays(cache, gs);
        const float4 m = __ldg(rmf + gs);
        int ok = sw_orientation_fast(R.r1, R.r2, make_float3(m.x, m.y, m.z), rec.d_q1, rec.d_q2);
        if (ok < 0) ok = sw_orientation_ok(views + q.tgt, sw_load_rays(rays, gs), rec.d_q1, rec.d_q2) ? 1 : 0;
        if (ok) { f |= 2; atomicAdd(csize + q.tgt_chunk_base + (long long)rec.tgt_seg * q.tgt_np + q.cy, 1); }
    }
    rflag[g] = f;
}

// region_off of every view = offset of its first chunk; written into the view table and a flat array (rank order is the
// order the chunk bases were assigned in, so the regions lie in processing order)
__global__ void __launch_bounds__(256)
k_sw_regions(int V, SwView* __restrict__ vt, const long long* __restrict__ cstart, long long num_chunks, const int* __restrict__ order,
             long long* __restrict__ region_by_rank)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > V) return;
    if (i == V) { region_by_rank[V] = cstart[num_chunks]; return; }
    const int v = order[i];
    const long long ro = cstart[vt[v].chunk_base];
    vt[v].region_off = ro;
    region_by_rank[i] = ro;
}

// P4: records -> entries of their chunk(s), in arbitrary order inside the chunk; key = what the chunk is sorted by
// (REF_GPU: the target segment of the list entry, sortMatchesByIDs commons.h:206-214; REF_CPU: the record index = append order)
__global__ void __launch_bounds__(256)
k_sw_scatter(const SwPairInfo* __restrict__ pinfo, const int* __restrict__ block_pair0, const l3d_match_rec* __restrict__ recs, int knn, long long slots,
             const unsigned char* __restrict__ rflag, const long long* __restrict__ cstart, int* __restrict__ ccur, uint2* __restrict__ e_kv, int cpu_sem)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= slots) return;
    const unsigned char f = rflag[g];
    if (!f) return;
    const unsigned int tseg = recs[g].tgt_seg;
    const long long row = g / knn;
    const SwPairInfo q = sw_pair_info(pinfo, block_pair0, row);
    const int r = (int)(row - q.row_off);
    if (f & 1) {
        const long long ch = q.src_chunk_base + (long long)r * q.src_np + q.cx;
        const long long x = cstart[ch] + atomicAdd(ccur + ch, 1);
        e_kv[x] = make_uint2(cpu_sem ? (unsigned int)g : tseg, (unsigned int)g);               // (sort key, record) in one 8-byte store
    }
    if (f & 2) {
        const long long ch = q.tgt_chunk_base + (long long)tseg * q.tgt_np + q.cy;
        const long long x = cstart[ch] + atomicAdd(ccur + ch, 1);
        e_kv[x] = make_uint2(cpu_sem ? (unsigned int)g : (unsigned int)r, (unsigned int)g | SW_INV);
    }
}

// P5: one warp per segment: every entry of the segment (all its chunks, contiguous) finds its place inside its chunk by counting
// the smaller keys (keys are unique inside a chunk), and is written in list order together with its initial flag (direct entries
// are active from the start) and, for inverse entries, the place its source will find it at.  Keys and chunk boundaries are read
// from shared-memory copies when the segment fits (n <= CS_MAXN, np <= CS_MAXNP), else straight from e_kv / cstart.
#define CS_WARPS 8
#define CS_MAXN 192
#define CS_MAXNP 64
__global__ void __launch_bounds__(32 * CS_WARPS)
k_sw_chunksort(const L3DViewDev* __restrict__ views, int V, long long N, const SwView* __restrict__ vt, const long long* __restrict__ cstart,
               const uint2* __restrict__ e_kv, unsigned int* __restrict__ e_val, unsigned char* __restrict__ e_flag, unsigned int* __restrict__ invpos)
{
    __shared__ unsigned int sk[CS_WARPS][CS_MAXN], sv[CS_WARPS][CS_MAXN];
    __shared__ int scb[CS_WARPS][CS_MAXNP + 1];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long gs = (long long)blockIdx.x * CS_WARPS + wid;
    if (gs >= N) return;
    const int lo = last_le(V, gs, [&](int i) { return views[i].seg_off; });
    const SwView me = vt[lo];
    const int np = me.np;
    if (np == 0) return;
    const long long ch0 = me.chunk_base + (gs - views[lo].seg_off) * np;
    const long long x0 = cstart[ch0], x1 = cstart[ch0 + np];
    const int n = (int)(x1 - x0);
    if (n == 0) return;
    const long long ro = me.region_off;
    // bound(c): start of chunk c relative to x0; key(i), val(i): entry i
    auto place = [&](auto bound, auto key, auto val) {
        for (int j = lane; j < n; j += 32) {
            const int cl = last_le(np, j, bound);
            const int a = bound(cl), b = bound(cl + 1);
            const unsigned int kj = key(j), vj = val(j);
            int rank = 0;
            for (int i = a; i < b; ++i) rank += key(i) < kj ? 1 : 0;
            const long long pos = x0 + a + rank;
            e_val[pos] = vj;
            if (vj & SW_INV) { e_flag[pos] = 0; invpos[vj & ~SW_INV] = (unsigned int)(pos - ro); }
            else e_flag[pos] = SW_ACTIVE;
        }
    };
    if (n <= CS_MAXN && np <= CS_MAXNP) {
        for (int c = lane; c <= np; c += 32) scb[wid][c] = (int)(cstart[ch0 + c] - x0);
        for (int j = lane; j < n; j += 32) { const uint2 kv = e_kv[x0 + j]; sk[wid][j] = kv.x; sv[wid][j] = kv.y; }
        __syncwarp();
        place([&](int c) { return scb[wid][c]; }, [&](int i) { return sk[wid][i]; }, [&](int i) { return sv[wid][i]; });
    } else {
        place([&](int c) { return (int)(cstart[ch0 + c] - x0); }, [&](int i) { return e_kv[x0 + i].x; }, [&](int i) { return e_kv[x0 + i].y; });
    }
}

// ---------------------------------------------------------------------------------------------- the chain kernel
// One CTA scores SW_SEGS consecutive segments of the view.  Their lists are contiguous in the match store, so the CTA stages
// ONE entry range [x0, x1) in shared memory, thread by thread (what scoringGPU's host pass, line3D.cc:1311-1355, and
// K_score_matches' prologue compute per match), compacts the indices of the active entries and then gives every active entry
// a thread that walks its own segment's list - K_score_matches' loop (cudawrapper.cu:304-359) - out of shared memory.
#ifndef SW_THREADS
#define SW_THREADS 256
#endif
#define SW_SEGS_MAX 16        // segments per CTA: chosen per view at launch time so that the view's CTAs are ONE resident wave
                              // (tools/sweep_score.py: 750 CTAs on 740 slots cost 20.7 ms per 1000 views, 600 CTAs 14.7 ms)
#define SW_CAP_MAX 4096       // list entries staged in shared memory per CTA, upper bound (longer ranges: global scratch)
#define SW_CAP_MAX_CPU 2048   // the same for REF_CPU

// staged entry: a = (depth1, depth2, target view or -1 if inactive, index of its chunk in the CTA), b = (dir.xyz, view to announce a
// positive score to or -1), r = (reg1, reg2) target regularisers, act = the ordered list of active entries; REF_CPU adds
// d64 = (double dir.xyz, length).  16 + 16 + 8 + 4 = 44 bytes, rounded up to 48 for the alignment of d64.
struct SwPtrs { float4* a; float4* b; float2* r; double4* d64; int* act; };
__host__ __device__ constexpr size_t sw_entry_bytes(bool cpu) { return cpu ? 48 + 32 : 48; }
// the arrays of `cap` staged entries from `base` (16-byte aligned): the shared-memory staging and the global scratch alike
__host__ __device__ __forceinline__ SwPtrs sw_carve(unsigned char* base, size_t cap, bool cpu)
{
    SwPtrs P;
    P.a = (float4*)base; P.b = P.a + cap; P.r = (float2*)(P.b + cap); P.act = (int*)(P.r + cap);
    P.d64 = cpu ? (double4*)(base + 48 * cap) : nullptr;
    return P;
}

// per-CTA tables: chunk boundaries of the CTA's segments, relative to the CTA's first entry (cb) and in the list of its active
// entries (cbA); what every chunk of the view points at (SwChunkInfo: other view, view to announce a positive score to or -1, the
// other view's k and double camera centre; built on the host); the rays of the segments.  The first two are held in shared memory
// up to these sizes and read from global memory beyond them - where they live is the only difference.
#define SW_MAXCH 512          // chunk boundaries held in shared memory (SW_SEGS * np + 1)
#define SW_MAXNP 64           // chunk descriptors held in shared memory
struct SwChunkInfo { int other, pub; float k; float pad; double Cx, Cy, Cz; };
struct SwSegInfo { float r1[3], r2[3]; double q1[3], q2[3]; };

struct SwScoreArgs {
    const float4* cache; const double* rays; const L3DViewDev* views; const l3d_match_rec* recs; int v;
    const SwView* vt; const SwChunkInfo* cinfo; const long long* cstart;
    const unsigned int* e_val; float* e_score; unsigned char* e_flag; const unsigned int* invpos;
    int* view_max_bits; int* M;
    unsigned char* gstage;          // global scratch (one view's region) for entry ranges longer than the shared-memory capacity
    int* gtab;                      // global scratch for cb, cbA of CTAs with more than SW_MAXCH chunks: 2 (nch + 1) ints per CTA
    float angle_reg, sim_t, q_thr, cos_thr;
    int segs, cap;                  // this launch: segments per CTA, staged entries per CTA (dynamic shared memory = sw_entry_bytes x cap)
};

// similarity of K_score_matches' inner loop (cudawrapper.cu:318-347) between the own entry and staged entry i, tests ordered
// cheapest first - the result is the same whichever of the three conditions rejects.
// Exact shortcut: sim = min(three terms), then truncated to 0 below sim_t.  If ONE term is certainly below sim_t the result is 0
// whatever the others are (fminf ignores NaN).  exp(-q) < sim_t is certain when q > q_thr = 1.01 * -ln(sim_t) (1 % margin >> the
// rounding of the division and of expf), and the angular term is certainly below sim_t when |cos| < cos_thr (same margin on the
// angle).  Everything inside the margins takes the full, reference-order path.
struct SwOwn { float d1, d2, pos_reg1, pos_reg2, thr1, thr2; float3 dir; };
__device__ __forceinline__ SwOwn sw_own(float4 ma, float4 mb, float2 rg, float k, float q_thr)
{
    SwOwn o;
    o.d1 = ma.x; o.d2 = ma.y;
    const float sig1 = k * o.d1, sig2 = k * o.d2;
    float pos_reg1 = 2.0f * sig1 * sig1, pos_reg2 = 2.0f * sig2 * sig2;
    const float pos_reg1_tgt = 2.0f * rg.x * rg.x, pos_reg2_tgt = 2.0f * rg.y * rg.y;
    o.pos_reg1 = 0.5f * (pos_reg1 + pos_reg1_tgt);
    o.pos_reg2 = 0.5f * (pos_reg2 + pos_reg2_tgt);
    o.thr1 = q_thr * o.pos_reg1; o.thr2 = q_thr * o.pos_reg2;
    o.dir = make_float3(mb.x, mb.y, mb.z);
    return o;
}
__device__ __forceinline__ float sw_sim(const SwOwn& o, const float4* __restrict__ sa, const float4* __restrict__ sb, int i, float angle_reg, float sim_t,
                                        float cos_thr)
{
    const float4 ta = sa[i];
    const float e1 = o.d1 - ta.x, e2 = o.d2 - ta.y;
    if (e1 * e1 > o.thr1 || e2 * e2 > o.thr2) return 0.0f;
    const float4 tb = sb[i];
    const float dp = o.dir.x * tb.x + o.dir.y * tb.y + o.dir.z * tb.z;
    if (fabsf(dp) < cos_thr) return 0.0f;
    const float angle = undirected_angle_deg(dp);
    const float sim_a = expf(-angle * angle / angle_reg);
    const float sim_p1 = expf(-e1 * e1 / o.pos_reg1), sim_p2 = expf(-e2 * e2 / o.pos_reg2);
    float sim = fminf(sim_a, fminf(sim_p1, sim_p2));
    if (sim < sim_t) sim = 0.0f;
    return sim;
}

// K_score_matches' accumulation (cudawrapper.cu:304-359) walks the segment's list and skips inactive entries and those of the own
// target camera.  Here it runs chunk by chunk over the ACTIVE entries only (ord = their indices in list order, cbA = chunk
// boundaries in that list).  A chunk is a run of entries with one target camera: its first entry flushes what the previous camera
// left pending (score += max(pending, sim); pending = 0), the others raise pending - exactly the reference's sequence of float
// additions, because the entries it skips contribute nothing (x + 0 == x) and a camera without active entries does not appear
// in the reference's list at all.
__device__ __forceinline__ float sw_score_gpu_chunks(const float4* __restrict__ sa, const float4* __restrict__ sb, float2 rg, const int* __restrict__ ord,
                                                     const int* __restrict__ cbA, const SwChunkInfo* __restrict__ cinfo, int c0, int np, int my_chunk, int me,
                                                     float k, float angle_reg, float sim_t, float q_thr, float cos_thr)
{
    const SwOwn o = sw_own(sa[me], sb[me], rg, k, q_thr);
    const int my_cam = __float_as_int(sa[me].z);
    float score3D = 0.0f, pending = 0.0f;
    int current_cam = -1;
    for (int c = 0; c < np; ++c) {
        const int cc = c0 + c;
        int t = cbA[cc];
        const int te = cbA[cc + 1];
        if (t == te || cc == my_chunk) continue;
        const int cam = cinfo[c].other;
        if (cam == my_cam) continue;
        if (cam != current_cam) {
            const float sim = sw_sim(o, sa, sb, ord[t], angle_reg, sim_t, cos_thr);
            pending = fmaxf(pending, sim);
            score3D += pending; pending = 0.0f; current_cam = cam;
            ++t;
        }
#pragma unroll 2
        for (; t < te; ++t) pending = fmaxf(pending, sw_sim(o, sa, sb, ord[t], angle_reg, sim_t, cos_thr));
    }
    score3D += pending;
    return score3D;
}

// scoringCPU (line3D.cc:1208-1294) + similarityForScoring (1417-1446) + angleBetweenSeg3D (1571-1583): the score is the sum
// over target cameras of the best similarity among that camera's matches, built with the reference's running update (add the
// first value of a camera, replace it when a larger one arrives) in list order; [lo, hi) indexes the ordered list of active
// entries ord.
#define SC_MAP 48
__device__ __forceinline__ float sw_score_cpu(const float4* __restrict__ sa, const double4* __restrict__ d64, float2 rg, const int* __restrict__ ord, int lo,
                                              int hi, int me, float k, float angle_reg, float sim_t)
{
    const float4 ma = sa[me];
    const int my_cam = __float_as_int(ma.z);
    const double4 D1 = d64[me];
    const float sig1 = ma.x * k, sig2 = ma.y * k;
    float reg1 = 2.0f * sig1 * sig1, reg2 = 2.0f * sig2 * sig2;
    reg1 = 0.5f * (reg1 + 2.0f * rg.x * rg.x); reg2 = 0.5f * (reg2 + 2.0f * rg.y * rg.y);
    auto sim_of = [&](int i) -> float {
        const double4 D2 = d64[i];
        if ((float)D1.w < L3D_EPS_D || (float)D2.w < L3D_EPS_D) return 0.0f;
        const float angle = undirected_angle_deg((float)(D1.x * D2.x + D1.y * D2.y + D1.z * D2.z));
        const float sim_a = expf(-angle * angle / angle_reg);
        const float4 d2 = sa[i];
        const float e1 = ma.x - d2.x, e2 = ma.y - d2.y;
        const float sim_p = fminf(expf(-e1 * e1 / reg1), expf(-e2 * e2 / reg2));
        const float sm = fminf(sim_a, sim_p);
        return sm > sim_t ? sm : 0.0f;
    };
    int cams[SC_MAP]; float best[SC_MAP]; int ncam = 0;
    float score3D = 0.0f;
    for (int t = lo; t < hi; ++t) {
        const int i = ord[t];
        const int cam = __float_as_int(sa[i].z);
        if (cam < 0 || cam == my_cam) continue;
        const float sim = sim_of(i);
        int slot = -1;
        for (int j = 0; j < ncam; ++j) if (cams[j] == cam) { slot = j; break; }
        if (slot >= 0) { if (sim > best[slot]) { score3D -= best[slot]; score3D += sim; best[slot] = sim; } }
        else if (ncam < SC_MAP) { score3D += sim; cams[ncam] = cam; best[ncam] = sim; ++ncam; }
        else {      // more target cameras than map slots: recover this camera's running maximum from the earlier entries
            bool seen = false; float cur = 0.0f;
            for (int u = lo; u < t; ++u) {
                const int j = ord[u];
                if (__float_as_int(sa[j].z) == cam) { const float sj = sim_of(j); if (!seen) { cur = sj; seen = true; } else if (sj > cur) cur = sj; }
            }
            if (seen) { if (sim > cur) { score3D -= cur; score3D += sim; } } else score3D += sim;
        }
    }
    return score3D;
}

// regularizers_tgt (line3D.cc:1350-1352) == View::regularizerFrom3Dpoint (view.cc:445-448): |P - C_tgt| * k_tgt in double, stored as
// float; REF_CPU also needs the double 3D segment (direction, float length) scoringCPU works on
template <bool CPU>
__device__ __forceinline__ float2 sw_target_reg(const L3DViewDev* V, const SwSegInfo& sg, float d1, float d2, const SwChunkInfo& ci, double4* d64_out)
{
    SegRaysQ Q;
    Q.r1 = d3(sg.q1[0], sg.q1[1], sg.q1[2]); Q.r2 = d3(sg.q2[0], sg.q2[1], sg.q2[2]); Q.rm = d3(0, 0, 0);
    D3 P1, P2;
    sw_unproject_pts(V, Q, d1, d2, &P1, &P2);
    const Seg3D S = seg3d(P1, P2);
    if (CPU) *d64_out = make_double4(S.dir.x, S.dir.y, S.dir.z, (double)S.length);
    const D3 Ct = d3(ci.Cx, ci.Cy, ci.Cz);
    return make_float2((float)(dnorm(dsub(S.P1, Ct)) * (double)ci.k), (float)(dnorm(dsub(S.P2, Ct)) * (double)ci.k));
}

template <bool CPU>
__device__ __forceinline__ void sw_score_range(const SwScoreArgs& A,const SwPtrs P, const int* __restrict__ cb, int* __restrict__ cbA,
                                               const SwChunkInfo* __restrict__ cinfo, const SwSegInfo* __restrict__ sinfo, int* __restrict__ wcnt,
                                               int nsegs, long long x0, int n)
{
    const L3DViewDev* V = A.views + A.v;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int np = A.vt[A.v].np;
    const int nch = nsegs * np;
    // ---- stage: a = (depth1, depth2, target view [inverse entries: -2 - view until they are known to be active], chunk index in the CTA)
    for (int j0 = 0; j0 < n; j0 += SW_THREADS) {
        const int j = j0 + threadIdx.x;
        if (j < n) {
            const long long x = x0 + j;
            const unsigned int val = A.e_val[x];
            const l3d_match_rec rec = A.recs[val & ~SW_INV];
            const int lo = last_le(nch, j, [&](int q) { return cb[q]; });          // chunk of entry j
            const int si = lo / np;
            const SwChunkInfo ci = cinfo[lo - si * np];
            const bool inv = (val & SW_INV) != 0u;
            const float d1 = inv ? rec.d_q1 : rec.d_p1, d2 = inv ? rec.d_q2 : rec.d_p2;
            const SwSegInfo& sg = sinfo[si];
            {   // D_unproject x2 + D_line_direction_3D (cudawrapper.cu:167-171, 40-43) with the cached float rays
                const float3 Cf = make_float3(V->C[0], V->C[1], V->C[2]);
                const float3 P1 = make_float3(Cf.x + d1 * sg.r1[0], Cf.y + d1 * sg.r1[1], Cf.z + d1 * sg.r1[2]);
                const float3 P2 = make_float3(Cf.x + d2 * sg.r2[0], Cf.y + d2 * sg.r2[1], Cf.z + d2 * sg.r2[2]);
                const float3 dir = normalize3(make_float3(P2.x - P1.x, P2.y - P1.y, P2.z - P1.z));
                // where a positive score has to be announced: the target view, if it is still to be processed (line3D.cc:1680)
                P.b[j] = make_float4(dir.x, dir.y, dir.z, __int_as_float(inv ? -1 : ci.pub));
            }
            if (!inv) P.r[j] = sw_target_reg<CPU>(V, sg, d1, d2, ci, CPU ? P.d64 + j : nullptr);      // inverse entries: only if they turn out active
            P.a[j] = make_float4(d1, d2, __int_as_float(inv ? -2 - ci.other : ci.other), __int_as_float(lo));
        }
    }
    // ---- everything above only read what the set-up kernels wrote: it may overlap the previous view's kernel (programmatic
    // dependent launch).  From here on the "active" bits that kernel publishes are needed.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    // active flags of the inverse entries + the ordered list of active entries (ord = P.act)
    int nact = 0;
    for (int j0 = 0; j0 < n; j0 += SW_THREADS) {
        const int j = j0 + threadIdx.x;
        bool active = false;
        if (j < n) {
            const float4 ma = P.a[j];
            const int cam = __float_as_int(ma.z);
            active = cam >= 0;
            if (!active) {
                const long long x = x0 + j;
                if (A.e_flag[x] & SW_ACTIVE) {
                    active = true;
                    const int lo = __float_as_int(ma.w), si = lo / np;
                    const SwChunkInfo ci = cinfo[lo - si * np];
                    P.a[j].z = __int_as_float(ci.other);
                    P.r[j] = sw_target_reg<CPU>(V, sinfo[si], ma.x, ma.y, ci, CPU ? P.d64 + j : nullptr);
                } else { P.a[j].z = __int_as_float(-1); A.e_score[x] = 0.0f; }
            }
        }
        const unsigned int bal = __ballot_sync(0xffffffffu, active);
        if (lane == 0) wcnt[wid] = __popc(bal);
        __syncthreads();
        int woff = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < SW_THREADS / 32; ++w) { const int cw = wcnt[w]; if (w < wid) woff += cw; tot += cw; }
        if (active) P.act[nact + woff + __popc(bal & ((1u << lane) - 1u))] = j;
        nact += tot;
        __syncthreads();
    }
    // chunk boundaries in the list of active entries
    for (int q = threadIdx.x; q <= nch; q += SW_THREADS) {
        const int bound = cb[q];
        int lo = 0, hi = nact;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (P.act[mid] < bound) lo = mid + 1; else hi = mid; }
        cbA[q] = lo;
    }
    __syncthreads();
    // ---- score the active entries, publish
    float vmax = 0.0f;
    for (int q = threadIdx.x; q < nact; q += SW_THREADS) {
        const int j = P.act[q];
        const int my_chunk = __float_as_int(P.a[j].w);
        const int si = my_chunk / np;
        const float k = __ldg(&A.views[A.v].k);     // re-read per entry: a register held across this loop spills vmax (REF_GPU)
        const float sc = CPU ? sw_score_cpu(P.a, P.d64, P.r[j], P.act, cbA[si * np], cbA[(si + 1) * np], j, k, A.angle_reg, A.sim_t)
                             : sw_score_gpu_chunks(P.a, P.b, P.r[j], P.act, cbA, cinfo, si * np, np, my_chunk, j, k, A.angle_reg, A.sim_t, A.q_thr, A.cos_thr);
        const long long x = x0 + j;
        const int T = __float_as_int(P.b[j].w);
        if (T >= 0 && sc > 0.0f) {      // storeInverseMatches; an inverse match that fails T's orientation check has no entry there
            const unsigned int ip = A.invpos[A.e_val[x]];
            if (ip != 0xFFFFFFFFu) A.e_flag[A.vt[T].region_off + ip] = SW_ACTIVE;
        }
        vmax = fmaxf(vmax, sc);
        A.e_score[x] = sc;
    }
    for (int o = 16; o; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (lane == 0 && vmax > 0.0f) atomicMax(A.view_max_bits + A.v, __float_as_int(vmax));
    // active entries per view.  Nothing reads them, but without this use of nact ptxas (CUDA 12.9, sm_90a) keeps the count in a
    // vector register instead of a uniform one and spills vmax in the scoring loop of both REF_GPU instantiations.
    if (threadIdx.x == 0 && nact) atomicAdd(A.M + A.v, nact);
}

// SMEM: the host knows that every CTA of the launch holds its chunk tables in shared memory, so the scoring loop addresses them as
// such (LDS, not generic loads); otherwise each CTA decides where its tables live.
template <bool CPU, bool SMEM>
__global__ void __launch_bounds__(SW_THREADS, CPU ? (SW_THREADS <= 256 ? 3 : 2) : (SW_THREADS <= 256 ? 5 : SW_THREADS <= 320 ? 4 : SW_THREADS <= 384 ? 3 : 2))
k_sw_score(const SwScoreArgs A)
{
    const int CAP = A.cap;
    asm volatile("griddepcontrol.launch_dependents;");       // the next view's kernel may start its independent part
    extern __shared__ __align__(16) unsigned char sw_smem[];
    __shared__ int cb_s[SW_MAXCH + 1], cbA_s[SW_MAXCH + 1];
    __shared__ SwChunkInfo cinfo_s[SW_MAXNP];
    __shared__ SwSegInfo sinfo[SW_SEGS_MAX];
    __shared__ int wcnt[SW_THREADS / 32];
    const L3DViewDev* V = A.views + A.v;
    const int s0 = blockIdx.x * A.segs;
    const int nsegs = min(A.segs, V->nseg - s0);
    const SwView me = A.vt[A.v];
    const int np = me.np, nch = nsegs * np;
    const long long chbase = me.chunk_base + (long long)s0 * np;
    const long long x0 = A.cstart[chbase];
    const int n = (int)(A.cstart[chbase + nch] - x0);
    if (n == 0) return;
    // where the tables and the staged entries live; the global ones are slices of scratch shared with the kernels of the
    // neighbouring views, so a CTA that uses them writes nothing before those kernels are done.  That includes cb: it could be
    // read from cstart before the wait instead, but then the staging would need a second look-up path.
    const bool cb_smem = SMEM || nch <= SW_MAXCH, ci_smem = SMEM || np <= SW_MAXNP, staged_smem = n <= CAP;
    int* const gtab = A.gtab + 2 * ((long long)s0 * np + blockIdx.x);
    int* cb = cb_smem ? cb_s : gtab;
    int* cbA = cb_smem ? cbA_s : gtab + nch + 1;
    const SwChunkInfo* cinfo = ci_smem ? cinfo_s : A.cinfo + me.ci_off;
    const SwPtrs P = staged_smem ? sw_carve(sw_smem, CAP, CPU) : sw_carve(A.gstage + sw_entry_bytes(CPU) * (x0 - me.region_off), n, CPU);
    if (!cb_smem || !staged_smem) asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int q = threadIdx.x; q <= nch; q += SW_THREADS) cb[q] = (int)(A.cstart[chbase + q] - x0);
    if (ci_smem) for (int c = threadIdx.x; c < np; c += SW_THREADS) cinfo_s[c] = A.cinfo[me.ci_off + c];
    if (threadIdx.x < nsegs) {
        const long long gs = V->seg_off + s0 + threadIdx.x;
        const SegRays R = load_rays(A.cache, gs);
        const SegRaysQ Q = sw_load_rays(A.rays, gs);
        SwSegInfo si;
        si.r1[0] = R.r1.x; si.r1[1] = R.r1.y; si.r1[2] = R.r1.z; si.r2[0] = R.r2.x; si.r2[1] = R.r2.y; si.r2[2] = R.r2.z;
        si.q1[0] = Q.r1.x; si.q1[1] = Q.r1.y; si.q1[2] = Q.r1.z; si.q2[0] = Q.r2.x; si.q2[1] = Q.r2.y; si.q2[2] = Q.r2.z;
        sinfo[threadIdx.x] = si;
    }
    __syncthreads();
    sw_score_range<CPU>(A, P, cb, cbA, cinfo, sinfo, wcnt, nsegs, x0, n);
}

void (*const l3d_sw_score_kernels[2][2])(SwScoreArgs) = {
    {k_sw_score<false, false>, k_sw_score<false, true>},
    {k_sw_score<true, false>, k_sw_score<true, true>},
};
size_t l3d_sw_score_smem_bytes(bool cpu_sem) { return sw_entry_bytes(cpu_sem) * (cpu_sem ? SW_CAP_MAX_CPU : SW_CAP_MAX); }

// ---------------------------------------------------------------------------------------------- after the chain
// filterMatches (line3D.cc:1586-1669) for every segment of every view: one thread per global segment
__global__ void __launch_bounds__(256)
k_sw_filter(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, int V, long long N, const SwView* __restrict__ vt,
            const long long* __restrict__ cstart, const unsigned int* __restrict__ e_val, const float* __restrict__ e_score,
            unsigned char* __restrict__ e_flag, const l3d_match_rec* __restrict__ recs, const int* __restrict__ view_max_bits, float min_best,
            float perc, int2* __restrict__ ranges, int* __restrict__ est_best /*per global seg: index of best match in the view region or -1*/,
            double* __restrict__ est_P)
{
    const long long gs = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gs >= N) return;
    const int lo = last_le(V, gs, [&](int i) { return views[i].seg_off; });
    const L3DViewDev* Vw = views + lo;
    const SwView me = vt[lo];
    const int s = (int)(gs - Vw->seg_off);
    const long long ch0 = me.chunk_base + (long long)s * me.np;
    const long long x0 = me.np ? cstart[ch0] : 0, x1 = me.np ? cstart[ch0 + me.np] : 0;
    long long best = -1;
    if (x1 > x0) {
        const float score_lim = perc * __int_as_float(view_max_bits[lo]);
        float best_score = 0.0f;
        for (long long x = x0; x < x1; ++x) {
            const unsigned char f = e_flag[x];
            if (!(f & SW_ACTIVE)) continue;
            const float sc = e_score[x];
            const bool keep = sc > 0.0f && sc > score_lim;
            if (keep) { e_flag[x] = f | SW_KEPT; if (sc > best_score) { best_score = sc; best = x; } }
        }
        if (!(best_score > min_best)) {
            best = -1;
            for (long long x = x0; x < x1; ++x) e_flag[x] &= (unsigned char)~SW_KEPT;
        }
        ranges[gs] = make_int2((int)(x0 - me.region_off), (int)(x1 - 1 - me.region_off));
    } else ranges[gs] = make_int2(-1, -1);
    est_best[gs] = best >= 0 ? (int)(best - me.region_off) : -1;
    if (best >= 0) {
        const float4 dep = sw_depths(e_val[best], recs);
        // unprojectMatch(best_match, true).  The rays are the ones k_sw_rays cached, recomputed from the 16-byte segment:
        // reading the 48 bytes of cached rays made this kernel 1.3 % slower on an H100 80GB HBM3 (700 W).
        const float4 sg = segs[gs];
        SegRaysQ q;
        q.r1 = dray(Vw->RtKinv_d, (double)sg.x, (double)sg.y); q.r2 = dray(Vw->RtKinv_d, (double)sg.z, (double)sg.w); q.rm = d3(0, 0, 0);
        D3 P1, P2;
        sw_unproject_pts(Vw, q, dep.x, dep.y, &P1, &P2);
        const Seg3D S3 = seg3d(P1, P2);
        double* o = est_P + 6 * gs;
        o[0] = S3.P1.x; o[1] = S3.P1.y; o[2] = S3.P1.z; o[3] = S3.P2.x; o[4] = S3.P2.y; o[5] = S3.P2.z;
    }
}

// the L3DPP::Match record of a decoded entry of view v
__device__ __forceinline__ l3d_match sw_match(const L3DViewDev* __restrict__ views, int v, const SwEntry& e, float score3D)
{
    l3d_match m;
    m.src_cam = views[v].cam_id; m.src_seg = (unsigned int)e.seg; m.tgt_cam = views[e.tgt_view].cam_id; m.tgt_seg = (unsigned int)e.tgt_seg;
    m.overlap = e.overlap; m.score3D = score3D; m.d_p1 = e.dep.x; m.d_p2 = e.dep.y; m.d_q1 = e.dep.z; m.d_q2 = e.dep.w;
    return m;
}

// the matches of one view as L3DPP::Match records (test / dump interface)
__global__ void __launch_bounds__(256)
k_sw_export(const L3DViewDev* __restrict__ views, int v, long long ro, int n, const L3DPairDev* __restrict__ pairs,
            const long long* __restrict__ row_off, int num_pairs, int knn, const l3d_match_rec* __restrict__ recs,
            const unsigned int* __restrict__ e_val, const float* __restrict__ e_score, const unsigned char* __restrict__ e_flag,
            unsigned char want, l3d_match* __restrict__ out, unsigned char* __restrict__ ok)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long x = ro + i;
    const bool take = (e_flag[x] & want) == want;
    ok[i] = take ? 1 : 0;
    if (!take) return;
    out[i] = sw_match(views, v, sw_decode(e_val[x], pairs, row_off, num_pairs, knn, recs), e_score[x]);
}

// compact list of the segments that have a 3D estimate: their best match (L3DPP::Match layout) and P1,P2
struct HasEstimate { __host__ __device__ long long operator()(int best) const { return best >= 0 ? 1ll : 0ll; } };
__global__ void __launch_bounds__(256)
k_collect_estimates(const L3DViewDev* __restrict__ views, int V, long long N, const SwView* __restrict__ vt,
                    const int* __restrict__ est_best, const long long* __restrict__ pos, const L3DPairDev* __restrict__ pairs,
                    const long long* __restrict__ row_off, int num_pairs, int knn, const l3d_match_rec* __restrict__ recs,
                    const unsigned int* __restrict__ e_val, const float* __restrict__ e_score, const double* __restrict__ est_P,
                    l3d_match* __restrict__ out_best, double* __restrict__ out_P)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    const int b = est_best[g];
    if (b < 0) return;
    const int lo = last_le(V, g, [&](int i) { return views[i].seg_off; });
    const long long x = vt[lo].region_off + b;     // an entry of segment g: its decoded segment is g - views[lo].seg_off
    const long long p = pos[g];
    out_best[p] = sw_match(views, lo, sw_decode(e_val[x], pairs, row_off, num_pairs, knn, recs), e_score[x]);
    for (int i = 0; i < 6; ++i) out_P[6 * p + i] = est_P[6 * g + i];
}

// ---------------------------------------------------------------------------------------------- host driver
// what the host knows of a sweep's layout that the steps after sweep_layout need
struct SweepLayout {
    std::vector<SwView> vt;     // per view: first chunk, chunk descriptors (region_off is written on the device)
    long long NC = 0;           // chunks of all views
    long long tab_max = 0;      // most chunk boundaries of one view's CTAs (nseg * np + CTAs): the chunk-table scratch
    long long nblocks = 0;      // blocks of the record-parallel set-up kernels
    long long Umax = 1;         // entries of the longest region: the long-list scratch (set by sweep_setup)
};

// The processing order, the chunk lists of every view and the tables of the set-up kernels, built on the host and uploaded; the
// buffers whose sizes follow from them reserved, and those the set-up kernels and the chain accumulate into cleared.
static int sweep_layout(l3d_ctx* c, SweepLayout& L)
{
    SweepState& S = c->sweep; cudaStream_t st = c->stream; int rc;
    const int V = c->num_views, NP = c->num_pairs;
    const long long slots = c->total_rows * c->knn;
    // processing order = ascending camID (std::map iteration, line3D.cc:704)
    S.order.resize(V);
    std::iota(S.order.begin(), S.order.end(), 0);
    std::stable_sort(S.order.begin(), S.order.end(), [&](int a, int b) { return c->h_views[a].cam_id < c->h_views[b].cam_id; });
    std::vector<int> rank(V);
    for (int i = 0; i < V; ++i) rank[S.order[i]] = i;
    // chunk descriptors of every view in list order: REF_GPU sorts a segment's matches by (tgt cam, tgt seg) (sortMatches,
    // line3D.cc:1196-1205): chunks by the other view's camID.  REF_CPU keeps the append order (scoringCPU does not sort): first
    // the inverse matches, stored by the earlier views in their processing order, then the direct ones in matching order.
    struct SwChunk { int pair, inv, other; };      // chunk c of a view: pair index, inverse?, the other view
    std::vector<std::vector<SwChunk> > chunks(V);
    for (int p = 0; p < NP; ++p) {
        const L3DPairDev& P = c->h_pairs[p];
        chunks[P.src].push_back(SwChunk{p, 0, P.tgt});
        if (rank[P.tgt] > rank[P.src]) chunks[P.tgt].push_back(SwChunk{p, 1, P.src});   // tgt still unprocessed when src stores its inverse matches (line3D.cc:1680)
    }
    std::vector<SwChunkInfo> cinfo; std::vector<SwView>& vt = L.vt; std::vector<int2> pairc(NP, make_int2(-1, -1));
    vt.assign(V, SwView{});
    for (int i = 0; i < V; ++i) {
        const int v = S.order[i];
        std::vector<SwChunk>& ch = chunks[v];
        if (c->semantics != L3D_SEM_REF_CPU) std::stable_sort(ch.begin(), ch.end(), [&](const SwChunk& a, const SwChunk& b) { return rank[a.other] != rank[b.other] ? rank[a.other] < rank[b.other] : a.inv > b.inv; });
        else std::stable_sort(ch.begin(), ch.end(), [&](const SwChunk& a, const SwChunk& b) {
            if (a.inv != b.inv) return a.inv > b.inv;
            return a.inv ? rank[a.other] < rank[b.other] : a.pair < b.pair; });
        vt[v].ci_off = (int)cinfo.size(); vt[v].np = (int)ch.size(); vt[v].chunk_base = L.NC;
        for (int k = 0; k < (int)ch.size(); ++k) {
            if (ch[k].inv) pairc[ch[k].pair].y = k; else pairc[ch[k].pair].x = k;
            const L3DViewDev& T = c->h_views[ch[k].other];
            // a positive score of a direct match is announced to the other view if that holds the inverse match (is processed later)
            const int pub = !ch[k].inv && rank[ch[k].other] > i ? ch[k].other : -1;
            cinfo.push_back(SwChunkInfo{ch[k].other, pub, T.k, 0.f, T.C_d[0], T.C_d[1], T.C_d[2]});
        }
        const long long nseg = c->h_views[v].nseg;
        L.NC += nseg * (long long)ch.size();
        L.tab_max = std::max(L.tab_max, nseg * ((long long)ch.size() + 1));
    }
    std::vector<long long> row_off(NP + 1);
    for (int p = 0; p < NP; ++p) row_off[p] = c->h_pairs[p].row_off;
    row_off[NP] = c->total_rows;
    std::vector<SwPairInfo> pinfo((size_t)NP + 1);
    for (int p = 0; p < NP; ++p) {
        const L3DPairDev& P = c->h_pairs[p];
        SwPairInfo& q = pinfo[p];
        q.row_off = row_off[p]; q.row_end = row_off[p + 1]; q.src = P.src; q.tgt = P.tgt;
        q.src_seg_off = c->h_views[P.src].seg_off; q.tgt_seg_off = c->h_views[P.tgt].seg_off;
        q.src_chunk_base = vt[P.src].chunk_base; q.tgt_chunk_base = vt[P.tgt].chunk_base; q.src_np = vt[P.src].np; q.tgt_np = vt[P.tgt].np;
        q.cx = pairc[p].x; q.cy = pairc[p].y;
    }
    { SwPairInfo& q = pinfo[NP]; std::memset(&q, 0, sizeof(q)); q.row_off = c->total_rows; q.row_end = (1ll << 62); q.cx = q.cy = -1; }   // sentinel
    L.nblocks = (slots + SW_SETUP_THREADS - 1) / SW_SETUP_THREADS;
    std::vector<int> bpair((size_t)std::max<long long>(L.nblocks, 1), 0);
    for (long long b = 0, p = 0; b < L.nblocks; ++b) {
        const long long row = (b * SW_SETUP_THREADS) / c->knn;
        while (p < NP && row >= row_off[p + 1]) ++p;          // pairs without rows are skipped
        bpair[b] = (int)p;
    }
    const long long NC = L.NC, N = c->total_segs;
    L3D_RESERVE(S.d_vt, sizeof(SwView) * (size_t)V, "view table"); L3D_RESERVE(S.d_cinfo, sizeof(SwChunkInfo) * cinfo.size(), "chunk descriptors");
    L3D_RESERVE(S.d_rowoff, 8 * (size_t)(NP + 1), "pair row offsets"); L3D_RESERVE(S.d_order, 4 * (size_t)V, "order"); L3D_RESERVE(S.d_region_off, 8 * (size_t)(V + 1), "region offsets");
    L3D_RESERVE(S.d_pinfo, sizeof(SwPairInfo) * (size_t)(NP + 1), "pair table"); L3D_RESERVE(S.d_bpair, 4 * bpair.size(), "first pair of every block");
    L3D_RESERVE(S.d_rays, 72 * N, "segment rays"); L3D_RESERVE(S.d_rmf, 16 * N, "mid-point rays"); L3D_RESERVE(S.d_rflag, slots, "record flags"); L3D_RESERVE(S.d_invpos, 4 * slots, "inverse positions");
    L3D_RESERVE(S.d_csize, 4 * (NC + 1), "chunk sizes"); L3D_RESERVE(S.d_ccur, 4 * (NC + 1), "chunk cursors"); L3D_RESERVE(S.d_cstart, 8 * (NC + 1), "chunk offsets");
    L3D_RESERVE(S.d_ranges, 8 * N, "ranges"); L3D_RESERVE(S.d_est_best, 4 * N, "estimates"); L3D_RESERVE(S.d_est_P, 48 * N, "estimate points");
    L3D_RESERVE(S.d_M, 4 * (size_t)V, "match counts"); L3D_RESERVE(S.d_vmax, 4 * (size_t)V, "view max");
    L3D_CUDA(c, cudaMemcpyAsync(S.d_vt.p, vt.data(), sizeof(SwView) * (size_t)V, cudaMemcpyHostToDevice, st), "view table");
    if (!cinfo.empty()) L3D_CUDA(c, cudaMemcpyAsync(S.d_cinfo.p, cinfo.data(), sizeof(SwChunkInfo) * cinfo.size(), cudaMemcpyHostToDevice, st), "chunk descriptors");
    L3D_CUDA(c, cudaMemcpyAsync(S.d_rowoff.p, row_off.data(), 8 * (size_t)(NP + 1), cudaMemcpyHostToDevice, st), "pair row offsets");
    L3D_CUDA(c, cudaMemcpyAsync(S.d_order.p, S.order.data(), 4 * (size_t)V, cudaMemcpyHostToDevice, st), "order");
    L3D_CUDA(c, cudaMemcpyAsync(S.d_pinfo.p, pinfo.data(), sizeof(SwPairInfo) * (size_t)(NP + 1), cudaMemcpyHostToDevice, st), "pair table");
    L3D_CUDA(c, cudaMemcpyAsync(S.d_bpair.p, bpair.data(), 4 * bpair.size(), cudaMemcpyHostToDevice, st), "first pair of every block");
    L3D_CUDA(c, cudaStreamSynchronize(st), "score sweep tables");      // cinfo / pinfo / bpair are locals
    L3D_CUDA(c, cudaMemsetAsync(S.d_csize.p, 0, 4 * (size_t)(NC + 1), st), "init chunk sizes");
    L3D_CUDA(c, cudaMemsetAsync(S.d_ccur.p, 0, 4 * (size_t)(NC + 1), st), "init chunk cursors");
    L3D_CUDA(c, cudaMemsetAsync(S.d_rflag.p, 0, (size_t)slots, st), "init record flags");
    L3D_CUDA(c, cudaMemsetAsync(S.d_invpos.p, 0xFF, 4 * (size_t)slots, st), "init inverse positions");   // "no inverse entry"
    L3D_CUDA(c, cudaMemsetAsync(S.d_M.p, 0, 4 * (size_t)V, st), "init counts");
    L3D_CUDA(c, cudaMemsetAsync(S.d_vmax.p, 0, 4 * (size_t)V, st), "init maxima");
    return L3D_OK;
}

// The match store: orientation flags of every record and the chunk sizes, chunk offsets and every view's region (downloaded: the
// chain's geometry and the size of the entry arrays follow from them), then the entries in list order.
static int sweep_setup(l3d_ctx* c, SweepLayout& L)
{
    SweepState& S = c->sweep; cudaStream_t st = c->stream; int rc;
    const int V = c->num_views, knn = c->knn;
    const long long slots = c->total_rows * knn, NC = L.NC, N = c->total_segs;
    const bool cpu_sem = c->semantics == L3D_SEM_REF_CPU;
    const L3DViewDev* views = c->views(); const l3d_match_rec* recs = (const l3d_match_rec*)c->d_recs.p;
    const unsigned int nbs = (unsigned int)L.nblocks;
    S.region_off.assign(V + 1, 0);
    if (c->num_pairs > 0 && slots > 0) {
        k_sw_rays<<<(unsigned int)((N + 255) / 256), 256, 0, st>>>(c->segs(), views, V, N, (double*)S.d_rays.p, (float4*)S.d_rmf.p);
        k_sw_flags<<<nbs, SW_SETUP_THREADS, 0, st>>>((const double*)S.d_rays.p, (const float4*)c->d_cache.p, (const float4*)S.d_rmf.p, views, (const SwPairInfo*)S.d_pinfo.p,
                                                     (const int*)S.d_bpair.p, (const int*)c->d_counts.p, recs, knn, slots, (unsigned char*)S.d_rflag.p, (int*)S.d_csize.p);
        if ((rc = l3d_cub(c, "chunk scan", [&](void* tmp, size_t& bytes) {
                 return cub::DeviceScan::ExclusiveSum(tmp, bytes, (const int*)S.d_csize.p, (long long*)S.d_cstart.p, NC + 1, st); }))) return rc;
        k_sw_regions<<<(V + 256) / 256, 256, 0, st>>>(V, (SwView*)S.d_vt.p, (const long long*)S.d_cstart.p, NC, (const int*)S.d_order.p, (long long*)S.d_region_off.p);
        L3D_CUDA(c, cudaMemcpyAsync(S.region_off.data(), S.d_region_off.p, 8 * (size_t)(V + 1), cudaMemcpyDeviceToHost, st), "region offsets");
        L3D_CUDA(c, cudaStreamSynchronize(st), "score sweep set-up");
        c->launches += 4;
    } else {
        L3D_CUDA(c, cudaMemsetAsync(S.d_cstart.p, 0, 8 * (size_t)(NC + 1), st), "chunk offsets");
        L3D_CUDA(c, cudaMemsetAsync(S.d_region_off.p, 0, 8 * (size_t)(V + 1), st), "region offsets");
    }
    const long long total = S.total = S.region_off[V];
    for (int i = 0; i < V; ++i) L.Umax = std::max(L.Umax, S.region_off[i + 1] - S.region_off[i]);
    if (L.Umax >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_score_sweep: view with more than 2^31 matches");
    L3D_RESERVE(S.d_eval, 4 * total, "entry records"); L3D_RESERVE(S.d_escore, 4 * total, "entry scores"); L3D_RESERVE(S.d_eflag, total, "entry flags");
    L3D_RESERVE(S.d_ekv, 8 * total, "unsorted entries");
    // global scratch of the chain, double-buffered (two kernels may be in flight): staged entries of the longest region, chunk
    // tables of the view with the most chunk boundaries
    L3D_RESERVE(S.d_gstage, 2 * sw_entry_bytes(cpu_sem) * L.Umax, "long-list scratch"); L3D_RESERVE(S.d_gtab, 2 * 2 * 4 * L.tab_max, "chunk table scratch");
    if (total > 0) {
        k_sw_scatter<<<nbs, SW_SETUP_THREADS, 0, st>>>((const SwPairInfo*)S.d_pinfo.p, (const int*)S.d_bpair.p, recs, knn, slots, (const unsigned char*)S.d_rflag.p,
                                                       (const long long*)S.d_cstart.p, (int*)S.d_ccur.p, (uint2*)S.d_ekv.p, cpu_sem ? 1 : 0);
        k_sw_chunksort<<<(unsigned int)((N + CS_WARPS - 1) / CS_WARPS), 32 * CS_WARPS, 0, st>>>(views, V, N, (const SwView*)S.d_vt.p, (const long long*)S.d_cstart.p,
                                                                                               (const uint2*)S.d_ekv.p, (unsigned int*)S.d_eval.p, (unsigned char*)S.d_eflag.p,
                                                                                               (unsigned int*)S.d_invpos.p);
        c->launches += 2;
    }
    return L3D_OK;
}

// Geometry of one view's chain launch (`entries` in its region, `nseg` segments): the fewest segments per CTA for which all CTAs
// are resident at once (one wave), or force_segs > 0 of them, and the entries each CTA stages in shared memory.
struct SwGeometry { int segs, cap; };
static SwGeometry sw_geometry(bool cpu_sem, long long entries, int nseg, int num_sms, int force_segs)
{
    const int cap_max = cpu_sem ? SW_CAP_MAX_CPU : SW_CAP_MAX;
    const int occ_regs = cpu_sem ? 3 : 5;               // resident CTAs per SM the register budget allows (launch bounds)
    const double avg = (double)entries / nseg;
    // staged entries: 45 % + 160 above the mean (a CTA whose range is longer falls back to the slow global-scratch path)
    auto cap_of = [&](int segs) { return std::min(cap_max, (int)((segs * avg * 1.45 + 160 + 63) / 64) * 64); };
    if (force_segs > 0) { const int segs = std::min(force_segs, SW_SEGS_MAX); return SwGeometry{segs, cap_of(segs)}; }
    SwGeometry g = {}; double best = 1e300;
    for (int segs = 1; segs <= SW_SEGS_MAX; ++segs) {
        const int cap = cap_of(segs);
        const int occ = std::max(1, std::min(occ_regs, (int)((227 * 1024) / (sw_entry_bytes(cpu_sem) * cap + 8500))));
        const long long ctas = (nseg + segs - 1) / segs;
        const double waves = std::ceil((double)ctas / ((double)num_sms * occ));
        const double cost = waves * (1.0 + segs * avg / SW_THREADS);      // waves x rounds of work per thread
        if (cost < best - 1e-9) { best = cost; g = SwGeometry{segs, cap}; }
    }
    return g;
}

// The chain: one k_sw_score launch per view with entries, in processing order.
static int sweep_chain(l3d_ctx* c, const SweepLayout& L, float two_sigA_sqr, float min_similarity)
{
    SweepState& S = c->sweep;
    if (S.total == 0) return L3D_OK;
    const bool cpu_sem = c->semantics == L3D_SEM_REF_CPU;
    // shortcut thresholds of sw_score_gpu (see there); disabled (never true) when sim_t <= 0 or the margins do not apply
    float q_thr = INFINITY, cos_thr = -1.0f;
    if (min_similarity > 0.0f && min_similarity < 1.0f) {
        q_thr = 1.01f * -std::log(min_similarity);
        const double ang = std::sqrt((double)q_thr * (double)two_sigA_sqr);           // degrees
        cos_thr = ang < 89.0 ? (float)(std::cos(ang * L3D_PI_D / 180.0) * (1.0 - 1e-4)) : -1.0f;
    }
    SwScoreArgs A = {};
    A.cache = (const float4*)c->d_cache.p; A.rays = (const double*)S.d_rays.p; A.views = c->views(); A.recs = (const l3d_match_rec*)c->d_recs.p;
    A.vt = (const SwView*)S.d_vt.p; A.cinfo = (const SwChunkInfo*)S.d_cinfo.p; A.cstart = (const long long*)S.d_cstart.p;
    A.e_val = (const unsigned int*)S.d_eval.p; A.e_score = (float*)S.d_escore.p; A.e_flag = (unsigned char*)S.d_eflag.p; A.invpos = (const unsigned int*)S.d_invpos.p;
    A.view_max_bits = (int*)S.d_vmax.p; A.M = (int*)S.d_M.p;
    A.angle_reg = two_sigA_sqr; A.sim_t = min_similarity; A.q_thr = q_thr; A.cos_thr = cos_thr;
    const size_t per_entry = sw_entry_bytes(cpu_sem);
    const int force_segs = getenv("L3D_SW_SEGS") ? atoi(getenv("L3D_SW_SEGS")) : 0;      // tools/sweep_score.py: override the geometry choice
    // programmatic dependent launch: a view's kernel may stage its lists while the previous view's kernel is still scoring (it waits
    // before it reads the bits that kernel publishes).  The first one follows ordinary kernels: plain stream order.
    cudaLaunchAttribute pdl;
    pdl.id = cudaLaunchAttributeProgrammaticStreamSerialization; pdl.val.programmaticStreamSerializationAllowed = 1;
    int launched = 0;
    for (int i = 0; i < c->num_views; ++i) {
        const int v = S.order[i], nseg = c->h_views[v].nseg;
        const long long entries = S.region_off[i + 1] - S.region_off[i];
        if (nseg == 0 || entries == 0) continue;
        const SwGeometry g = sw_geometry(cpu_sem, entries, nseg, c->num_sms, force_segs);
        A.v = v; A.segs = g.segs; A.cap = g.cap;
        A.gstage = (unsigned char*)S.d_gstage.p + (launched & 1) * per_entry * L.Umax;     // double-buffered scratch
        A.gtab = (int*)S.d_gtab.p + (launched & 1) * 2 * L.tab_max;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned int)((nseg + g.segs - 1) / g.segs)); cfg.blockDim = dim3(SW_THREADS); cfg.dynamicSmemBytes = per_entry * (size_t)g.cap;
        cfg.stream = c->stream; cfg.attrs = &pdl; cfg.numAttrs = launched ? 1 : 0;
        const bool smem_tables = L.vt[v].np <= SW_MAXNP && g.segs * L.vt[v].np <= SW_MAXCH;
        L3D_CUDA(c, cudaLaunchKernelEx(&cfg, l3d_sw_score_kernels[cpu_sem][smem_tables], A), "k_sw_score");
        ++launched; ++c->launches;
    }
    L3D_CUDA(c, cudaGetLastError(), "score sweep launch");
    return L3D_OK;
}

// filterMatches and the best 3D estimate of every segment for all views, then the estimates compacted on the device: flags ->
// exclusive scan -> gather (best match record + P1,P2)
static int sweep_filter(l3d_ctx* c, float min_best_score, float min_best_perc)
{
    SweepState& S = c->sweep; cudaStream_t st = c->stream; int rc;
    const int V = c->num_views; const long long N = c->total_segs;
    const SwView* vt = (const SwView*)S.d_vt.p; const l3d_match_rec* recs = (const l3d_match_rec*)c->d_recs.p;
    const unsigned int* e_val = (const unsigned int*)S.d_eval.p; const float* e_score = (const float*)S.d_escore.p;
    S.n_est = 0;
    if (N == 0) return L3D_OK;
    const unsigned int nb = (unsigned int)((N + 255) / 256);
    k_sw_filter<<<nb, 256, 0, st>>>(c->segs(), c->views(), V, N, vt, (const long long*)S.d_cstart.p, e_val, e_score, (unsigned char*)S.d_eflag.p, recs,
                                    (const int*)S.d_vmax.p, min_best_score, min_best_perc, (int2*)S.d_ranges.p, (int*)S.d_est_best.p, (double*)S.d_est_P.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_sw_filter");
    L3D_RESERVE(S.d_est_pos, 8 * (size_t)(N + 1), "estimate positions");
    cub::TransformInputIterator<long long, HasEstimate, const int*> flags((const int*)S.d_est_best.p, HasEstimate());
    ScanTotal t;
    if ((rc = l3d_scan_total(c, flags, (long long*)S.d_est_pos.p, N, (const int*)S.d_est_best.p, t, "estimate scan"))) return rc;
    L3D_CUDA(c, cudaStreamSynchronize(st), "score sweep");
    S.n_est = t.last_out + HasEstimate()(t.last_src);
    L3D_RESERVE(S.d_est_out_best, sizeof(l3d_match) * (size_t)std::max<long long>(S.n_est, 1), "estimate records");
    L3D_RESERVE(S.d_est_out_P, 48 * (size_t)std::max<long long>(S.n_est, 1), "estimate points");
    if (S.n_est > 0) {
        k_collect_estimates<<<nb, 256, 0, st>>>(c->views(), V, N, vt, (const int*)S.d_est_best.p, (const long long*)S.d_est_pos.p, (const L3DPairDev*)c->d_pairs.p,
                                                (const long long*)S.d_rowoff.p, c->num_pairs, c->knn, recs, e_val, e_score, (const double*)S.d_est_P.p,
                                                (l3d_match*)S.d_est_out_best.p, (double*)S.d_est_out_P.p);
        c->launches += 3;
        L3D_CUDA(c, cudaGetLastError(), "k_collect_estimates");
    }
    return L3D_OK;
}

extern "C" {

int l3d_score_sweep(l3d_ctx* c, float two_sigA_sqr, float min_similarity, float min_best_score, float min_best_perc)
{
    if (!c) return L3D_ERR_INVALID;
    c->drop(Stage::Sweep);
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_score_sweep: call l3d_match_pairs first");
    cudaSetDevice(c->device);
    if (c->total_rows * c->knn >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_score_sweep: more than 2^31 match slots");
    SweepState& S = c->sweep; SweepLayout L; int rc;
    if ((rc = sweep_layout(c, L))) return rc;
    // device time of the three phases: set-up, chain, filter + estimates
    ScopedEvent ev[4];
    for (ScopedEvent& e : ev) if ((rc = e.create(c))) return rc;
    cudaEventRecord(ev[0].e, c->stream);
    if ((rc = sweep_setup(c, L))) return rc;
    cudaEventRecord(ev[1].e, c->stream);
    if ((rc = sweep_chain(c, L, two_sigA_sqr, min_similarity))) return rc;
    cudaEventRecord(ev[2].e, c->stream);
    if ((rc = sweep_filter(c, min_best_score, min_best_perc))) return rc;
    cudaEventRecord(ev[3].e, c->stream);
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "score sweep");
    cudaEventElapsedTime(&S.ms_setup, ev[0].e, ev[1].e); cudaEventElapsedTime(&S.ms_chain, ev[1].e, ev[2].e); cudaEventElapsedTime(&S.ms_filter, ev[2].e, ev[3].e);
    if (getenv("L3D_SWEEP_TIMING")) fprintf(stderr, "[l3d] score sweep: set-up %.3f ms, chain %.3f ms (%d views), filter+estimates %.3f ms\n", S.ms_setup, S.ms_chain, c->num_views, S.ms_filter);
    S.valid = true;
    return L3D_OK;
}

// matches of one view after scoring, in the reference's list order (REF_GPU: segment, then tgt cam, tgt seg).
// kept_only != 0: only the matches that survived filterMatches.  Returns the number of matches (even if > cap).
long long l3d_get_view_matches(l3d_ctx* c, int view, int kept_only, l3d_match* out, long long cap)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->sweep.valid) return l3d_fail(c, L3D_ERR_STATE, "l3d_get_view_matches: call l3d_score_sweep first");
    if (view < 0 || view >= c->num_views) return l3d_fail(c, L3D_ERR_INVALID, "l3d_get_view_matches: view out of range");
    cudaSetDevice(c->device);
    SweepState& S = c->sweep;
    const int i = (int)(std::find(S.order.begin(), S.order.end(), view) - S.order.begin());
    const long long ro = S.region_off[i];
    const int n = (int)(S.region_off[i + 1] - ro);
    if (n == 0) return 0;
    int rc;
    L3D_RESERVE(S.d_export, sizeof(l3d_match) * (size_t)n, "export records");
    L3D_RESERVE(S.d_export_ok, (size_t)n, "export flags");
    k_sw_export<<<(n + 255) / 256, 256, 0, c->stream>>>(c->views(), view, ro, n, (const L3DPairDev*)c->d_pairs.p, (const long long*)S.d_rowoff.p, c->num_pairs, c->knn,
                                                     (const l3d_match_rec*)c->d_recs.p, (const unsigned int*)S.d_eval.p, (const float*)S.d_escore.p,
                                                     (const unsigned char*)S.d_eflag.p, (unsigned char)(kept_only ? (SW_ACTIVE | SW_KEPT) : SW_ACTIVE),
                                                     (l3d_match*)S.d_export.p, (unsigned char*)S.d_export_ok.p);
    std::vector<l3d_match> m(n); std::vector<unsigned char> ok(n);
    L3D_CUDA(c, cudaMemcpyAsync(m.data(), S.d_export.p, sizeof(l3d_match) * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "download");
    L3D_CUDA(c, cudaMemcpyAsync(ok.data(), S.d_export_ok.p, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "download");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    long long cnt = 0;
    for (int x = 0; x < n; ++x) {
        if (!ok[x]) continue;
        if (out && cnt < cap) out[cnt] = m[x];
        ++cnt;
    }
    return cnt;
}

// best-match 3D estimates (estimated_position3D_, line3D.cc:1635-1647), compacted on the device by k_collect_estimates
// at the end of the sweep, in global segment order (view index, segment).
long long l3d_get_estimates(l3d_ctx* c, l3d_match* best_out, double* p1p2_out, long long cap)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->sweep.valid) return l3d_fail(c, L3D_ERR_STATE, "l3d_get_estimates: call l3d_score_sweep first");
    cudaSetDevice(c->device);
    SweepState& S = c->sweep;
    const long long n = S.n_est;
    if (n == 0 || n > cap) return n;
    if (best_out) L3D_CUDA(c, cudaMemcpyAsync(best_out, S.d_est_out_best.p, sizeof(l3d_match) * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "download estimates");
    if (p1p2_out) L3D_CUDA(c, cudaMemcpyAsync(p1p2_out, S.d_est_out_P.p, 48 * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "download estimates");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    return n;
}

} // extern "C"
