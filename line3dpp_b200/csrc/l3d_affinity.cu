// l3d_affinity.cu — pairwise affinities between 3D hypotheses and the replicator-dynamics diffusion.
//
//   l3d_affinity_matrix : computingAffinityMatrix (line3D.cc:1852-1979), which the reference runs on the host under three
//                       mutexes, in five steps: the kept matches in emission order; their candidates - Line3D::similarity
//                       (line3D.cc:1467-1553) above min_affinity and, with collinearity links, the links through target and
//                       source (1904-1974) - counted per kept match (k_aff_count), scanned and written in the reference's order
//                       (k_aff_fill); unused() as a fixpoint over a stable pair sort; local ids by first appearance; the CLEdge list.
//   l3d_rdd           : replicator_dynamics_diffusion_GPU (cudawrapper.cu:708-766) on CSR/CSC SoA arrays instead of two
//                       AoS float4 COO copies: 20 B/nnz/iteration of compulsory traffic instead of >= 64.  The arithmetic
//                       (positional lock-step product, per-row sequential sums, clamps) is kept operation for operation,
//                       so the result is bit-identical to the reference kernels; the linear search for the transposed
//                       slot (cudawrapper.cu:524-542) is replaced by a precomputed permutation.
#include "l3d_cub.cuh"
#include "l3d_device_f64.cuh"
#include "l3d_sweep.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <algorithm>
#include <cstdlib>
#include <vector>

// Line3D::similarity(s1, m1, seg2, truncate = false) (line3D.cc:1467-1553) for two segments that both have a 3D estimate:
// P1/P2 = their estimates (6 doubles each), m1/m2 = depths of their best matches, v1/v2 = their views
__device__ __forceinline__ float aff_similarity(const L3DViewDev* v1, const L3DViewDev* v2, const double* P1, const double* P2, float4 m1, float4 m2,
                                                float two_sigA_sqr, float med_scene_depth_lines)
{
    const Seg3D s1 = seg3d(d3(P1[0], P1[1], P1[2]), d3(P1[3], P1[4], P1[5]));
    const Seg3D s2 = seg3d(d3(P2[0], P2[1], P2[2]), d3(P2[3], P2[4], P2[5]));
    if (s1.length < L3D_EPS_D || s2.length < L3D_EPS_D) return 0.0f;
    const float angle = undirected_angle_deg((float)ddot(s1.dir, s2.dir));         // angleBetweenSeg3D (line3D.cc:1571-1583)
    float sim_a = expf(-angle * angle / two_sigA_sqr);
    float cutoff1 = v1->median_depth, cutoff2 = v2->median_depth;
    if (med_scene_depth_lines > L3D_EPS_D) { cutoff1 = fminf(cutoff1, med_scene_depth_lines); cutoff2 = fminf(cutoff2, med_scene_depth_lines); }
    float d11 = dist_p2l(s2, s1.P1), d12 = dist_p2l(s2, s1.P2), d21 = dist_p2l(s1, s2.P1), d22 = dist_p2l(s1, s2.P2);
    float sig11 = m1.x > cutoff1 ? cutoff1 * v1->k : m1.x * v1->k;
    float sig12 = m1.y > cutoff1 ? cutoff1 * v1->k : m1.y * v1->k;
    float reg11 = 2.0f * sig11 * sig11, reg12 = 2.0f * sig12 * sig12;
    float sig21 = m2.x > cutoff2 ? cutoff2 * v2->k : m2.x * v2->k;
    float sig22 = m2.y > cutoff2 ? cutoff2 * v2->k : m2.y * v2->k;
    float reg21 = 2.0f * sig21 * sig21, reg22 = 2.0f * sig22 * sig22;
    float sim_p1 = fminf(expf(-d11 * d11 / reg11), expf(-d12 * d12 / reg12));
    float sim_p2 = fminf(expf(-d21 * d21 / reg21), expf(-d22 * d22 / reg22));
    return fminf(sim_a, fminf(sim_p1, sim_p2));
}

// everything a thread needs to read the sweep's match store (l3d_sweep.cuh)
struct SwStore {
    const SwView* vt; const L3DPairDev* pairs; const long long* row_off; int num_pairs, knn; const l3d_match_rec* recs;
    const unsigned int* e_val; const unsigned char* e_flag;
};
// depths of the best match of global segment g (its estimate), b = est_best[g]
__device__ __forceinline__ float4 sw_best_depths(const SwStore& M, int view, int b) { return sw_depths(M.e_val[M.vt[view].region_off + b], M.recs); }

// Parameters of the candidate kernels.  kx[0, K) are the kept matches in emission order: regions in processing order, each one
// segment-major (l3d_sweep.cuh), so the kept matches of a segment are consecutive and lie within its ranges[] entry.
struct AffArgs {
    const L3DViewDev* views; const int* order; const long long* region_off; int V;     // order, region_off: per processing rank
    SwStore M;
    const int* est_best; const double* est_P; const int2* ranges;
    const long long* kx; long long K;
    const long long* cptr; const int* cidx;             // collinear lists, CSR over global segments; null: links off
    float two_sigA_sqr, med_scene_depth_lines, min_affinity;
};

// kept match q: source segment gi in view v1, target gj in view v2, their similarity if both have an estimate, and whether it
// exceeds min_affinity
struct AffMatch { int v1, v2; long long gi, gj; float sim; bool pass; };
__device__ __forceinline__ AffMatch aff_match(const AffArgs& a, long long q)
{
    const long long x = a.kx[q];
    const SwEntry me = sw_decode(a.M.e_val[x], a.M.pairs, a.M.row_off, a.M.num_pairs, a.M.knn, a.M.recs);
    AffMatch m;
    m.v1 = a.order[last_le(a.V, x, [&](int i) { return a.region_off[i]; })];          // the view whose region contains x
    m.v2 = me.tgt_view;
    m.gi = a.views[m.v1].seg_off + me.seg; m.gj = a.views[m.v2].seg_off + me.tgt_seg;
    const int b1 = a.est_best[m.gi], b2 = a.est_best[m.gj];
    m.sim = 0.0f; m.pass = false;
    if (b1 >= 0 && b2 >= 0) {
        m.sim = aff_similarity(a.views + m.v1, a.views + m.v2, a.est_P + 6 * m.gi, a.est_P + 6 * m.gj, sw_best_depths(a.M, m.v1, b1),
                               sw_best_depths(a.M, m.v2, b2), a.two_sigA_sqr, a.med_scene_depth_lines);
        m.pass = m.sim > a.min_affinity;
    }
    return m;
}

// The links of estimate gs (view v1) through segment g of view v: the segments collinear with g that have an estimate and a
// similarity with gs above min_affinity, in list order (line3D.cc:1904-1937 with g the target, 1941-1974 with g = gs).
// emit(g2, sim) for each; returns their number.
template <class Emit>
__device__ __forceinline__ int aff_links(const AffArgs& a, int v1, long long gs, int v, long long g, Emit&& emit)
{
    const long long k0 = a.cptr[g], k1 = a.cptr[g + 1];
    if (k0 == k1) return 0;
    const float4 m1 = sw_best_depths(a.M, v1, a.est_best[gs]);
    const L3DViewDev* vg = a.views + v;
    int n = 0;
    for (long long k = k0; k < k1; ++k) {
        const long long g2 = vg->seg_off + a.cidx[k];
        const int b2 = a.est_best[g2];
        if (b2 < 0) continue;
        const float s = aff_similarity(a.views + v1, vg, a.est_P + 6 * gs, a.est_P + 6 * g2, m1, sw_best_depths(a.M, v, b2), a.two_sigA_sqr,
                                       a.med_scene_depth_lines);
        if (s > a.min_affinity) { emit(g2, s); ++n; }
    }
    return n;
}

// The links through source gi (view v1) follow kept match q's events if q is gi's last kept match and one of gi's kept matches
// passed: passed(p) for p = q, q - 1, ... down to gi's first.
template <class Passed>
__device__ __forceinline__ bool aff_source_links_after(const AffArgs& a, long long q, int v1, long long gi, Passed&& passed)
{
    const long long ro = a.M.vt[v1].region_off;
    const int2 r = a.ranges[gi];
    if (q + 1 < a.K && a.kx[q + 1] <= ro + r.y) return false;
    for (long long p = q; p >= 0 && a.kx[p] >= ro + r.x; --p)
        if (passed(p)) return true;
    return false;
}

// Candidates, count: one thread per kept match writes its similarity, segments and pass flag and, with links, its number of
// events: the direct edge and the links through the target if it passes, then the links through the source if aff_source_links_after.
// Without links the pass flag is the count.  LINKS == (a.cptr != null), a template argument so that the instantiation without links
// has only the registers it needs (76, as many as the similarity alone; 96 with links).
template <bool LINKS>
__global__ void __launch_bounds__(256)
k_aff_count(const AffArgs a, float* __restrict__ sim, int* __restrict__ flag, long long* __restrict__ gi, long long* __restrict__ gj,
            int* __restrict__ cnt)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= a.K) return;
    const AffMatch m = aff_match(a, q);
    sim[q] = m.sim; flag[q] = m.pass ? 1 : 0; gi[q] = m.gi; gj[q] = m.gj;
    if (!LINKS) return;
    const auto none = [](long long, float) {};
    int n = m.pass ? 1 + aff_links(a, m.v1, m.gi, m.v2, m.gj, none) : 0;
    if (aff_source_links_after(a, q, m.v1, m.gi, [&](long long p) { return p == q ? m.pass : aff_match(a, p).pass; }))
        n += aff_links(a, m.v1, m.gi, m.v1, m.gi, none);
    cnt[q] = n;
}

// Candidates, fill: kept match q writes its events from evptr[q] on, in k_aff_count's order, and with links each one's parent:
// -1 the direct edge, >= 0 the direct edge a link through the target belongs to, -2 "some direct edge of my source".
template <bool LINKS>
__global__ void __launch_bounds__(256)
k_aff_fill(const AffArgs a, const float* __restrict__ sim, const int* __restrict__ flag, const long long* __restrict__ gi,
           const long long* __restrict__ gj, const long long* __restrict__ evptr, long long* __restrict__ out_i, long long* __restrict__ out_j,
           float* __restrict__ out_w, int* __restrict__ out_par)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= a.K || (!LINKS && !flag[q])) return;
    const long long g = gi[q], e0 = evptr[q];
    long long e = e0;
    const auto put = [&](long long j, float w, int par) { out_i[e] = g; out_j[e] = j; out_w[e] = w; if (LINKS) out_par[e] = par; ++e; };
    const auto view_of = [&](long long s) { return last_le(a.V, s, [&](int i) { return a.views[i].seg_off; }); };
    const int v1 = view_of(g);
    if (flag[q]) {
        put(gj[q], sim[q], -1);
        if (LINKS) aff_links(a, v1, g, view_of(gj[q]), gj[q], [&](long long g2, float s) { put(g2, s, (int)e0); });
    }
    if (LINKS && aff_source_links_after(a, q, v1, g, [&](long long p) { return flag[p] != 0; }))
        aff_links(a, v1, g, v1, g, [&](long long g2, float s) { put(g2, s, -2); });
}

// ================================================================================================ diffusion
__global__ void __launch_bounds__(256)
k_rdd_keys(long long nnz, const int* __restrict__ ei, const int* __restrict__ ej, unsigned long long* __restrict__ krow,
           unsigned long long* __restrict__ kcol, unsigned int* __restrict__ idx)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    krow[e] = ((unsigned long long)(unsigned int)ei[e] << 32) | (unsigned int)ej[e];
    kcol[e] = ((unsigned long long)(unsigned int)ej[e] << 32) | (unsigned int)ei[e];
    idx[e] = (unsigned int)e;
}
// gather sorted values + row/col of each entry, mark row (or col) starts
__global__ void __launch_bounds__(256)
k_rdd_gather(long long nnz, const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ idx,
             const float* __restrict__ w, float* __restrict__ val, int* __restrict__ major, int* __restrict__ minor)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    const unsigned long long k = keys[e];
    const int ma = (int)(k >> 32), mi = (int)(k & 0xFFFFFFFFull);
    val[e] = w[idx[e]]; major[e] = ma; minor[e] = mi;
}
// CSR/CSC pointers: ptr[r] = first sorted position whose major index is >= r (r = 0..n), by binary search
__global__ void __launch_bounds__(256) k_rdd_ptr(int n, int nnz, const int* __restrict__ major, int* __restrict__ ptr)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n) return;
    int lo = 0, hi = nnz;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (major[mid] < r) lo = mid + 1; else hi = mid; }
    ptr[r] = lo;
}
// transposed slot of every row-sorted entry (a,b): first position of (b,a) in row b, -1 if absent
__global__ void __launch_bounds__(256)
k_rdd_tslot(long long nnz, const int* __restrict__ prow, const int* __restrict__ pcol, const int* __restrict__ rowptr, int* __restrict__ tslot)
{
    const long long y = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= nnz) return;
    const int a = prow[y], b = pcol[y];
    int lo = rowptr[b], hi = rowptr[b + 1];
    const int end = hi;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (pcol[mid] < a) lo = mid + 1; else hi = mid; }
    tslot[y] = (lo < end && pcol[lo] == a) ? lo : -1;
}
// ---- sector-aligned rows ----------------------------------------------------------------------------------------------
// The lock-step walk reads a run of P.row(r) and a run of W.col(c) per entry.  With 4-byte loads every thread of a warp
// touches a different 128-byte line on every step (one L1 wavefront per thread and step: the first version was bound by
// exactly that).  Values are therefore kept in PADDED arrays whose rows/columns start on 32-byte boundaries (rp4/cp4 =
// start in float4 units, always even; rows padded with zeros to a multiple of 8); the walk loads float4 and still adds
// the products strictly in k order, so the sums round exactly like the reference's.
__global__ void __launch_bounds__(256) k_rdd_len4(int n, const int* __restrict__ ptr, int* __restrict__ len4)
{
    // rows padded to a multiple of EIGHT floats: every row starts on a 32-byte sector boundary, so the back-to-back float4
    // loads of a walk use whole sectors (with 16-byte alignment half of every gathered sector was wasted L2 bandwidth)
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) len4[r] = 2 * ((ptr[r + 1] - ptr[r] + 7) >> 3);
}
__global__ void __launch_bounds__(256) k_rdd_pad(long long nnz, const int* __restrict__ major, const int* __restrict__ ptr, const int* __restrict__ p4,
                                                 const float* __restrict__ val, float* __restrict__ padded)
{
    const long long y = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= nnz) return;
    const int r = major[y];
    padded[4ll * p4[r] + (y - ptr[r])] = val[y];
}
__global__ void __launch_bounds__(256) k_rdd_unpad(long long nnz, const int* __restrict__ major, const int* __restrict__ ptr, const int* __restrict__ p4,
                                                   const float* __restrict__ padded, float* __restrict__ val)
{
    const long long y = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= nnz) return;
    const int r = major[y];
    val[y] = padded[4ll * p4[r] + (y - ptr[r])];
}
// per-entry walk descriptors, built once (the structure is constant over the iterations): everything the step needs is
// then read with coalesced 16-byte loads instead of eight dependent scattered pointer look-ups per entry
//   x = first float4 of P.row(r)   y = first float4 of W.col(c)   z = walk length min(len_r, len_c)   w = own padded slot
// and dst = padded slot of the transposed entry P'(r,c) (or -1)
__global__ void __launch_bounds__(256)
k_rdd_plan(long long nnz, const int* __restrict__ prow, const int* __restrict__ pcol, const int* __restrict__ rowptr, const int* __restrict__ colptr,
           const int* __restrict__ rp4, const int* __restrict__ cp4, const int* __restrict__ tslot, int4* __restrict__ plan, int* __restrict__ dst)
{
    const long long y = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= nnz) return;
    const int c = prow[y], r = pcol[y];                 // "transpose" (cudawrapper.cu:493-495)
    const int rs = rowptr[r], m = min(rowptr[r + 1] - rs, colptr[c + 1] - colptr[c]);
    plan[y] = make_int4(rp4[r], cp4[c], m, 4 * rp4[c] + (int)(y - rowptr[c]));
    const int t = tslot[y];
    dst[y] = t >= 0 ? 4 * rp4[r] + (t - rs) : -1;
}
// K_sparseMat_diffusion_step (cudawrapper.cu:480-544) on the padded arrays: entry y = (a,b) of P produces P'(b,a).
// One thread per entry, walking in steps of EIGHT values = one whole 32-byte sector of P.row(b) and of W.col(a) per step
// (two back-to-back 16-byte loads of the same sector each; sm_90 has no 32-byte load); the first two steps are in flight
// together, which is the memory-level parallelism this latency-bound gather needs at 5 resident CTAs per SM.  No per-element
// guards: beyond the walk length min(len_r, len_c) at least one of the two factors lies in its row's zero padding (rows are
// padded to 8), the product is +0 and `mul + 0 == mul` exactly, so every entry still accumulates exactly the reference's
// products in the reference's k order (weights and P are finite).
#ifndef RDD_MINB
#define RDD_MINB 5
#endif
struct __align__(32) F8 { float v[8]; };
__device__ __forceinline__ F8 ld256(const float* p)
{
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    F8 r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}
__global__ void __launch_bounds__(256, RDD_MINB)
k_rdd_step8(long long nnz, const int4* __restrict__ plan, const int* __restrict__ dst, const float* __restrict__ Pp, const float* __restrict__ Wp,
            float* __restrict__ Pnp)
{
    const long long y = (long long)blockIdx.x * 256 + threadIdx.x;
    if (y >= nnz) return;
    const int4 pl = plan[y];
    const int d = dst[y];
    const int n8 = (pl.z + 7) >> 3;
    const float* pr = Pp + 4ll * pl.x;
    const float* wc = Wp + 4ll * pl.y;
    // the first two steps (16 values: most walks) are requested together, before anything waits on them
    F8 p0, w0, p1, w1;
    if (n8 > 0) { p0 = ld256(pr); w0 = ld256(wc); }
    if (n8 > 1) { p1 = ld256(pr + 8); w1 = ld256(wc + 8); }
    const float own = (pl.z > 0 || d >= 0) ? Pp[pl.w] : 0.0f;
    float m = 0.0f;
    if (n8 > 0) {
#pragma unroll
        for (int e = 0; e < 8; ++e) m += p0.v[e] * w0.v[e];
    }
    if (n8 > 1) {
#pragma unroll
        for (int e = 0; e < 8; ++e) m += p1.v[e] * w1.v[e];
    }
    for (int k8 = 2; k8 < n8; ++k8) {
        const F8 pv = ld256(pr + 8 * k8), wv = ld256(wc + 8 * k8);
#pragma unroll
        for (int e = 0; e < 8; ++e) m += pv.v[e] * wv.v[e];
    }
    m *= own;                                           // times P(a,b) itself
    if (m < L3D_EPS_F) m = L3D_EPS_F;
    if (d >= 0) Pnp[d] = m;
}
// K_sparseMat_row_normalization (cudawrapper.cu:432-477), 4 lanes per row, one float4 each per pass: coalesced loads and
// stores, and the row sum is still added strictly in slot order - the running sum is handed from lane to lane (lane j adds
// its four values to what lane j-1 produced).  No guards: padding slots hold +0 (x + 0 == x exactly, 0 / sum == 0).
__global__ void __launch_bounds__(256)
k_rdd_normalize_q(int n, const int* __restrict__ rowptr, const int* __restrict__ rp4, float* __restrict__ Pp)
{
    // control flow is kept warp-uniform (trip count = the longest of the warp's 8 rows, no early exit) so that the shuffles can
    // name the full warp: sub-warp masks compile to a WARPSYNC / collective sequence per shuffle, which made the first version
    // of this kernel instruction-bound
    const int lane = threadIdx.x & 31, gl = lane & 3, g0 = lane & ~3;
    const long long r = ((long long)blockIdx.x * 256 + threadIdx.x) >> 2;
    const int len = r < n ? rowptr[r + 1] - rowptr[r] : 0;
    const int n4 = 2 * ((len + 7) >> 3);                 // float4 per padded row (k_rdd_len4)
    float4* row = reinterpret_cast<float4*>(Pp) + (r < n ? rp4[r] : 0);
    const int n4max = __reduce_max_sync(0xffffffffu, n4);
    float sum = 0.0f;
    float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f);         // this lane's float4 of the first chunk (rows of <= 16 values are done from it)
    for (int c0 = 0; c0 < n4max; c0 += 4) {
        const float4 v = c0 + gl < n4 ? row[c0 + gl] : make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 == 0) v0 = v;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float t = sum; t += v.x; t += v.y; t += v.z; t += v.w;          // what lane j of the group contributes, in slot order
            sum = __shfl_sync(0xffffffffu, t, g0 + j);
        }
    }
    if (len == 0) return;
    if (sum < L3D_EPS_F) sum = L3D_EPS_F;
    // padding slots hold 0: 0 / sum is 0, but a zero dividend sends the IEEE divide down its slow path (FCHK), which made 52 % of
    // this kernel's instructions - skip them
#define RDD_DIV(x) if (x != 0.0f) { asm volatile(""); x = x / sum; }      /* the empty asm keeps the branch from being if-converted */
    if (n4 <= 4) { if (gl < n4) { RDD_DIV(v0.x) RDD_DIV(v0.y) RDD_DIV(v0.z) RDD_DIV(v0.w) row[gl] = v0; } }
    else for (int c = gl; c < n4; c += 4) { float4 w = row[c]; RDD_DIV(w.x) RDD_DIV(w.y) RDD_DIV(w.z) RDD_DIV(w.w) row[c] = w; }
#undef RDD_DIV
}

__global__ void __launch_bounds__(256) k_iota(long long n, unsigned int* __restrict__ idx)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (unsigned int)i;
}

// ---- affinity matrix bookkeeping on the device (see l3d_affinity_matrix) ----------------------------------------
static int bits_i64(long long n) { int b = 1; while ((1ll << b) < n) ++b; return b; }
__global__ void __launch_bounds__(256) k_aff_keys(long long ne, const long long* __restrict__ gi, const long long* __restrict__ gj,
                                                  unsigned long long* __restrict__ key, unsigned int* __restrict__ val)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    const unsigned long long a = (unsigned long long)min(gi[e], gj[e]), b = (unsigned long long)max(gi[e], gj[e]);
    key[e] = (a << 32) | b; val[e] = (unsigned int)e;
}
// unused() with conditional events (line3D.cc:1881-1974): event e enters A_ iff its parent did (direct events have none)
// and no EARLIER event of the same unordered pair did.  All dependencies point to earlier events, so iterating
//   acc[e] = parent_ok(e, acc_prev) && no earlier event e' of the same pair with parent_ok(e', acc_prev)
// from acc = 0 reaches the sequential answer after (longest dependency chain) rounds and then stays.  Without
// collinearity links every event is direct and the first round is already final (head of every run of the stable sort).
__device__ __forceinline__ bool aff_parent_ok(int e, const int* __restrict__ par, const long long* __restrict__ gi, const int* __restrict__ acc_prev,
                                              const int* __restrict__ found_prev)
{
    if (!par) return true;
    const int p = par[e];
    return p == -1 ? true : p >= 0 ? acc_prev[p] != 0 : found_prev[gi[e]] != 0;
}
__global__ void __launch_bounds__(256)
k_aff_round(long long ne, const unsigned long long* __restrict__ key, const unsigned int* __restrict__ val, const int* __restrict__ par,
            const long long* __restrict__ gi, const int* __restrict__ acc_prev, const int* __restrict__ found_prev, int* __restrict__ acc_new,
            int* __restrict__ changed)
{
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ne) return;
    const int e = (int)val[j];
    bool a = aff_parent_ok(e, par, gi, acc_prev, found_prev);
    const unsigned long long k = key[j];
    for (long long jj = j - 1; a && jj >= 0 && key[jj] == k; --jj)          // stable sort: earlier position = earlier in emission order
        if (aff_parent_ok((int)val[jj], par, gi, acc_prev, found_prev)) a = false;
    acc_new[e] = a ? 1 : 0;
    if ((acc_prev[e] != 0) != a) *changed = 1;
}
// found_aff of every source segment (line3D.cc:1900): some DIRECT event of it was accepted
__global__ void __launch_bounds__(256)
k_aff_found(long long ne, const int* __restrict__ par, const long long* __restrict__ gi, const int* __restrict__ acc, int* __restrict__ found)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < ne && acc[e] && par[e] == -1) found[gi[e]] = 1;
}
__global__ void __launch_bounds__(256) k_aff_time(long long ne, const int* __restrict__ keep, const long long* __restrict__ q, const long long* __restrict__ gi,
                                                  const long long* __restrict__ gj, unsigned long long* __restrict__ time)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne || !keep[e]) return;
    atomicMin(time + gi[e], 2ull * (unsigned long long)q[e]);          // id1 is looked up before id2 (line3D.cc:1884-1887)
    atomicMin(time + gj[e], 2ull * (unsigned long long)q[e] + 1ull);
}
__global__ void __launch_bounds__(256) k_aff_nodeflags(long long N, const unsigned long long* __restrict__ time, int* __restrict__ flag)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < N) flag[g] = time[g] != ~0ull;
}
__global__ void __launch_bounds__(256) k_aff_nodes(long long N, const int* __restrict__ flag, const long long* __restrict__ pos, const unsigned long long* __restrict__ time,
                                                   unsigned long long* __restrict__ key, unsigned int* __restrict__ val)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N || !flag[g]) return;
    key[pos[g]] = time[g]; val[pos[g]] = (unsigned int)g;
}
__global__ void __launch_bounds__(256) k_aff_ids(long long n, const unsigned int* __restrict__ seg_sorted, int* __restrict__ id_of, long long* __restrict__ l2g)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    id_of[seg_sorted[i]] = (int)i; l2g[i] = (long long)seg_sorted[i];
}
__global__ void __launch_bounds__(256) k_aff_emit(long long ne, const int* __restrict__ keep, const long long* __restrict__ q, const long long* __restrict__ gi,
                                                  const long long* __restrict__ gj, const float* __restrict__ w, const int* __restrict__ id_of,
                                                  int* __restrict__ ei, int* __restrict__ ej, float* __restrict__ ew)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne || !keep[e]) return;
    const long long o = 2 * q[e];
    const int a = id_of[gi[e]], b = id_of[gj[e]];
    ei[o] = a; ej[o] = b; ew[o] = w[e];
    ei[o + 1] = b; ej[o + 1] = a; ew[o + 1] = w[e];
}

struct KeptFlag { const unsigned char* f; __host__ __device__ int operator()(long long x) const { return (f[x] & SW_KEPT) ? 1 : 0; } };

// ---- the steps of l3d_affinity_matrix; l3d_affinity_edges takes the first two ----------------------------------------------------
// the kept matches (filterMatches survivors) in emission order into A.d_kx: everything below works on this list, not on the whole
// match store (2.5e9 entries at BASELINE configs[4])
static int kept_list(l3d_ctx* c, long long* n_kept)
{
    SweepState& S = c->sweep; AffinityState& A = c->aff; cudaStream_t st = c->stream; int rc;
    const long long total = S.total, BLK = 1ll << 30; long long K = 0;
    DevBuf& d_cnt = A.d_evptr;               // scratch for the counts until the candidates write the event offsets
    L3D_RESERVE(d_cnt, 16, "kept count");
    std::vector<long long> kept_in_block;
    for (long long base = 0; base < total; base += BLK) {
        const int nblk = (int)std::min(BLK, total - base);
        cub::CountingInputIterator<long long> idx(base);
        cub::TransformInputIterator<int, KeptFlag, cub::CountingInputIterator<long long> > flags(idx, KeptFlag{(const unsigned char*)S.d_eflag.p});
        if ((rc = l3d_cub(c, "kept count", [&](void* tmp, size_t& bytes) { return cub::DeviceReduce::Sum(tmp, bytes, flags, (int*)d_cnt.p, nblk, st); }))) return rc;
        int cnt = 0;
        L3D_CUDA(c, cudaMemcpyAsync(&cnt, d_cnt.p, 4, cudaMemcpyDeviceToHost, st), "kept count");
        L3D_CUDA(c, cudaStreamSynchronize(st), "kept count");
        kept_in_block.push_back(cnt); K += cnt;
    }
    *n_kept = K;
    if (K == 0) return L3D_OK;
    L3D_RESERVE(A.d_kx, 8 * K, "kept list");
    long long done = 0; size_t bi = 0;
    for (long long base = 0; base < total; base += BLK, ++bi) {
        const int nblk = (int)std::min(BLK, total - base);
        if (kept_in_block[bi] == 0) continue;
        cub::CountingInputIterator<long long> idx(base);
        cub::TransformInputIterator<int, KeptFlag, cub::CountingInputIterator<long long> > flags(idx, KeptFlag{(const unsigned char*)S.d_eflag.p});
        if ((rc = l3d_cub(c, "kept list", [&](void* tmp, size_t& bytes) {
                 return cub::DeviceSelect::Flagged(tmp, bytes, idx, flags, (long long*)A.d_kx.p + done, (int*)d_cnt.p, nblk, st); }))) return rc;
        done += kept_in_block[bi];
    }
    c->launches += 2 * (long long)kept_in_block.size();
    return L3D_OK;
}

// The kept matches with sim > min_affinity and, with collinearity links on, their links (line3D.cc:1904-1974): the candidates in
// emission order into A.d_aff_oi / oj / ow (and their parents into A.d_aff_par), by count, one scan, fill.  Returns their number (or < 0).
static long long affinity_candidates(l3d_ctx* c, float two_sigA_sqr, float med_scene_depth_lines, float min_affinity)
{
    SweepState& S = c->sweep; AffinityState& A = c->aff; const CollinState& CL = c->collin; cudaStream_t st = c->stream; int rc;
    const int V = c->num_views; long long K = 0;
    if ((rc = kept_list(c, &K)) || K == 0) return rc;
    L3D_RESERVE(A.d_aff_sim, 4 * K, "affinity sims"); L3D_RESERVE(A.d_aff_flag, 4 * K, "affinity flags");
    L3D_RESERVE(A.d_aff_gi, 8 * K, "affinity gi"); L3D_RESERVE(A.d_aff_gj, 8 * K, "affinity gj"); L3D_RESERVE(A.d_evptr, 8 * K, "event offsets");
    if (CL.valid) L3D_RESERVE(A.d_aff_cnt, 4 * K, "event counts");
    // S.d_order and S.d_region_off are the sweep's: it uploads the order and writes the region offsets, and nothing changes them until
    // the next sweep
    const AffArgs a = {c->views(), (const int*)S.d_order.p, (const long long*)S.d_region_off.p, V,
                       {(const SwView*)S.d_vt.p, (const L3DPairDev*)c->d_pairs.p, (const long long*)S.d_rowoff.p, c->num_pairs, c->knn,
                        (const l3d_match_rec*)c->d_recs.p, (const unsigned int*)S.d_eval.p, (const unsigned char*)S.d_eflag.p},
                       (const int*)S.d_est_best.p, (const double*)S.d_est_P.p, (const int2*)S.d_ranges.p, (const long long*)A.d_kx.p, K,
                       CL.valid ? (const long long*)CL.d_ptr.p : nullptr, CL.valid ? (const int*)CL.d_idx.p : nullptr,
                       two_sigA_sqr, med_scene_depth_lines, min_affinity};
    const unsigned int nb = (unsigned int)((K + 255) / 256);
    float* sim = (float*)A.d_aff_sim.p; int* flag = (int*)A.d_aff_flag.p; long long* gi = (long long*)A.d_aff_gi.p; long long* gj = (long long*)A.d_aff_gj.p;
    int* cnt = CL.valid ? (int*)A.d_aff_cnt.p : flag;        // links off: an event per passing kept match
    (CL.valid ? k_aff_count<true> : k_aff_count<false>)<<<nb, 256, 0, st>>>(a, sim, flag, gi, gj, cnt);
    ++c->launches;
    ScanTotal t;
    if ((rc = l3d_scan_total(c, (const int*)cnt, (long long*)A.d_evptr.p, K, cnt, t, "event scan"))) return rc;
    c->launches += 2;
    L3D_CUDA(c, cudaStreamSynchronize(st), "affinity events");
    const long long ne = t.last_out + t.last_src;
    if (ne == 0) return 0;
    if (ne >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "affinity: more than 2^31 candidate events");
    L3D_RESERVE(A.d_aff_oi, 8 * ne, "edges i"); L3D_RESERVE(A.d_aff_oj, 8 * ne, "edges j"); L3D_RESERVE(A.d_aff_ow, 4 * ne, "edges w");
    if (CL.valid) L3D_RESERVE(A.d_aff_par, 4 * ne, "edge parents");
    (CL.valid ? k_aff_fill<true> : k_aff_fill<false>)<<<nb, 256, 0, st>>>(a, sim, flag, gi, gj, (const long long*)A.d_evptr.p, (long long*)A.d_aff_oi.p,
                                                                        (long long*)A.d_aff_oj.p, (float*)A.d_aff_ow.p, (int*)A.d_aff_par.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_aff_fill");
    return ne;
}

// unused() (line3D.cc:1982-2002) into A.d_keep: the candidates stably sorted by unordered segment pair, then the fixpoint over the
// conditional events (see k_aff_round)
static int unused_fixpoint(l3d_ctx* c, long long ne)
{
    AffinityState& A = c->aff; const long long N = c->total_segs; cudaStream_t st = c->stream; int rc;
    const unsigned int nbe = (unsigned int)((ne + 255) / 256); const long long* oi = (const long long*)A.d_aff_oi.p;
    L3D_RESERVE(A.d_key, 8 * ne, "pair keys"); L3D_RESERVE(A.d_key2, 8 * ne, "pair keys"); L3D_RESERVE(A.d_val, 4 * ne, "pair vals"); L3D_RESERVE(A.d_val2, 4 * ne, "pair vals");
    L3D_RESERVE(A.d_keep, 4 * ne, "keep flags"); L3D_RESERVE(A.d_keep2, 4 * ne, "keep flags"); L3D_RESERVE(A.d_found, 4 * N, "found flags"); L3D_RESERVE(A.d_changed, 16, "changed flag");
    k_aff_keys<<<nbe, 256, 0, st>>>(ne, oi, (const long long*)A.d_aff_oj.p, (unsigned long long*)A.d_key.p, (unsigned int*)A.d_val.p);
    ++c->launches;
    if ((rc = l3d_cub(c, "pair sort", [&](void* tmp, size_t& bytes) {
             return cub::DeviceRadixSort::SortPairs(tmp, bytes, (const unsigned long long*)A.d_key.p, (unsigned long long*)A.d_key2.p, (const unsigned int*)A.d_val.p,
                                                    (unsigned int*)A.d_val2.p, (int)ne, 0, 32 + bits_i64(N), st); }))) return rc;
    c->launches += 8;
    // without collinearity links every event is direct: one round, the head of every run of the sort
    const int* par = c->collin.valid ? (const int*)A.d_aff_par.p : nullptr;
    L3D_CUDA(c, cudaMemsetAsync(A.d_keep.p, 0, 4 * ne, st), "clear keep");
    L3D_CUDA(c, cudaMemsetAsync(A.d_found.p, 0, 4 * N, st), "clear found");
    int* acc_prev = (int*)A.d_keep.p; int* acc_new = (int*)A.d_keep2.p;
    for (int round = 0;; ++round) {
        if (round > 100000) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_affinity_matrix: unused() fixpoint did not converge");
        L3D_CUDA(c, cudaMemsetAsync(A.d_changed.p, 0, 4, st), "clear changed");
        k_aff_round<<<nbe, 256, 0, st>>>(ne, (const unsigned long long*)A.d_key2.p, (const unsigned int*)A.d_val2.p, par, oi,
                                         acc_prev, (const int*)A.d_found.p, acc_new, (int*)A.d_changed.p);
        std::swap(acc_prev, acc_new);
        ++c->launches;
        if (!par) break;
        L3D_CUDA(c, cudaMemsetAsync(A.d_found.p, 0, 4 * N, st), "clear found");
        k_aff_found<<<nbe, 256, 0, st>>>(ne, par, oi, acc_prev, (int*)A.d_found.p);
        ++c->launches;
        int changed = 0;
        L3D_CUDA(c, cudaMemcpyAsync(&changed, A.d_changed.p, 4, cudaMemcpyDeviceToHost, st), "changed flag");
        L3D_CUDA(c, cudaStreamSynchronize(st), "affinity fixpoint");
        if (!changed) break;
    }
    if (acc_prev != (int*)A.d_keep.p) L3D_CUDA(c, cudaMemcpyAsync(A.d_keep.p, acc_prev, 4 * ne, cudaMemcpyDeviceToDevice, st), "keep flags");
    return L3D_OK;
}

// getLocalID (line3D.cc:2005-2023): A.d_q = position of every accepted candidate among the accepted ones (A.K of them), local ids
// in order of first appearance, the source of an edge before its target (A.d_idof, A.d_l2g, A.n_ids of them)
static int local_ids(l3d_ctx* c, long long ne)
{
    AffinityState& A = c->aff; const long long N = c->total_segs; cudaStream_t st = c->stream; int rc;
    const unsigned int nbe = (unsigned int)((ne + 255) / 256), nbn = (unsigned int)((N + 255) / 256);
    L3D_RESERVE(A.d_q, 8 * (ne + 1), "edge positions"); L3D_RESERVE(A.d_time, 8 * N, "appearance times");
    L3D_RESERVE(A.d_nflag, 4 * N, "node flags"); L3D_RESERVE(A.d_npos, 8 * (N + 1), "node positions"); L3D_RESERVE(A.d_idof, 4 * N, "id of segment");
    if ((rc = l3d_cub(c, "edge scan", [&](void* tmp, size_t& bytes) {
             return cub::DeviceScan::ExclusiveSum(tmp, bytes, (const int*)A.d_keep.p, (long long*)A.d_q.p, ne, st); }))) return rc;
    c->launches += 2;
    L3D_CUDA(c, cudaMemsetAsync(A.d_time.p, 0xFF, 8 * N, st), "init times");
    k_aff_time<<<nbe, 256, 0, st>>>(ne, (const int*)A.d_keep.p, (const long long*)A.d_q.p, (const long long*)A.d_aff_oi.p, (const long long*)A.d_aff_oj.p,
                                    (unsigned long long*)A.d_time.p);
    k_aff_nodeflags<<<nbn, 256, 0, st>>>(N, (const unsigned long long*)A.d_time.p, (int*)A.d_nflag.p);
    c->launches += 2;
    ScanTotal edges, nodes;         // both totals under one synchronisation
    if ((rc = l3d_scan_total(c, (const int*)A.d_nflag.p, (long long*)A.d_npos.p, N, (const int*)A.d_nflag.p, nodes, "node scan"))) return rc;
    c->launches += 2;
    if ((rc = l3d_read_total(c, (const long long*)A.d_q.p, (const int*)A.d_keep.p, ne, edges, "edge count"))) return rc;
    L3D_CUDA(c, cudaStreamSynchronize(st), "affinity matrix");
    A.K = edges.last_out + edges.last_src; A.n_ids = nodes.last_out + nodes.last_src;
    L3D_RESERVE(A.d_nkey, 8 * A.n_ids, "node keys"); L3D_RESERVE(A.d_nkey2, 8 * A.n_ids, "node keys"); L3D_RESERVE(A.d_nval, 4 * A.n_ids, "node vals");
    L3D_RESERVE(A.d_nval2, 4 * A.n_ids, "node vals"); L3D_RESERVE(A.d_l2g, 8 * A.n_ids, "local2global");
    k_aff_nodes<<<nbn, 256, 0, st>>>(N, (const int*)A.d_nflag.p, (const long long*)A.d_npos.p, (const unsigned long long*)A.d_time.p, (unsigned long long*)A.d_nkey.p, (unsigned int*)A.d_nval.p);
    ++c->launches;
    if ((rc = l3d_cub(c, "node sort", [&](void* tmp, size_t& bytes) {
             return cub::DeviceRadixSort::SortPairs(tmp, bytes, (const unsigned long long*)A.d_nkey.p, (unsigned long long*)A.d_nkey2.p, (const unsigned int*)A.d_nval.p,
                                                    (unsigned int*)A.d_nval2.p, (int)A.n_ids, 0, 64, st); }))) return rc;
    c->launches += 8;
    k_aff_ids<<<(unsigned int)((A.n_ids + 255) / 256), 256, 0, st>>>(A.n_ids, (const unsigned int*)A.d_nval2.p, (int*)A.d_idof.p, (long long*)A.d_l2g.p);
    ++c->launches;
    return L3D_OK;
}

// the CLEdge list: (id1, id2, w), (id2, id1, w) per accepted edge, in emission order
static int emit_edges(l3d_ctx* c, long long ne)
{
    AffinityState& A = c->aff; int rc;
    L3D_RESERVE(A.d_ei, 4 * 2 * A.K, "A i"); L3D_RESERVE(A.d_ej, 4 * 2 * A.K, "A j"); L3D_RESERVE(A.d_ew, 4 * 2 * A.K, "A w");
    k_aff_emit<<<(unsigned int)((ne + 255) / 256), 256, 0, c->stream>>>(ne, (const int*)A.d_keep.p, (const long long*)A.d_q.p, (const long long*)A.d_aff_oi.p,
                                                                      (const long long*)A.d_aff_oj.p, (const float*)A.d_aff_ow.p, (const int*)A.d_idof.p,
                                                                      (int*)A.d_ei.p, (int*)A.d_ej.p, (float*)A.d_ew.p);
    ++c->launches;
    return L3D_OK;
}

extern "C" {

// Affinity edges between segments with 3D estimates, in the reference's emission order (estimate order, then match
// list order), BEFORE the "unused" de-duplication and local-id assignment (line3D.cc:1881-1900).
// out_gi/out_gj are GLOBAL segment indices (view seg offset + seg id in l3d_set_views order).  Returns the count.
long long l3d_affinity_edges(l3d_ctx* c, float two_sigA_sqr, float med_scene_depth_lines, float min_affinity,
                             long long* out_gi, long long* out_gj, float* out_w, long long cap)
{
    if (!c) return L3D_ERR_INVALID;
    if (!(min_affinity >= 0.0f)) { c->drop(Stage::Affinity); return l3d_fail(c, L3D_ERR_INVALID, "l3d_affinity_edges: min_affinity must be >= 0"); }
    if (!c->sweep.valid) return l3d_fail(c, L3D_ERR_STATE, "l3d_affinity_edges: call l3d_score_sweep first");
    cudaSetDevice(c->device);
    const AffinityState& A = c->aff;
    const long long ne = affinity_candidates(c, two_sigA_sqr, med_scene_depth_lines, min_affinity);
    if (ne <= 0 || !out_gi || ne > cap) return ne;
    cudaStream_t st = c->stream;
    L3D_CUDA(c, cudaMemcpyAsync(out_gi, A.d_aff_oi.p, 8 * (size_t)ne, cudaMemcpyDeviceToHost, st), "download edges");
    L3D_CUDA(c, cudaMemcpyAsync(out_gj, A.d_aff_oj.p, 8 * (size_t)ne, cudaMemcpyDeviceToHost, st), "download edges");
    L3D_CUDA(c, cudaMemcpyAsync(out_w, A.d_aff_ow.p, 4 * (size_t)ne, cudaMemcpyDeviceToHost, st), "download edges");
    L3D_CUDA(c, cudaStreamSynchronize(st), "affinity download");
    return ne;
}

// The complete affinity matrix A_ of computingAffinityMatrix (line3D.cc:1852-1979) built on the device: candidates as
// above, then the reference's bookkeeping reproduced with sorts instead of mutex-protected maps:
//   unused(i,j)   (line3D.cc:1982-2002): of all candidates of an unordered segment pair only the FIRST in emission order
//                 survives                      -> stable radix sort by pair key, keep the head of every run;
//   getLocalID    (line3D.cc:2005-2023): ids in order of first appearance (source of an accepted edge before its target)
//                                               -> atomicMin of the appearance time per segment, sort segments by it.
// Output: the CLEdge list in the reference's order, (id1,id2,w),(id2,id1,w) per accepted edge, and local2global as
// global segment indices.  Returns the number of list entries (2 per edge), even if > cap_edges (then nothing is copied).
long long l3d_affinity_matrix(l3d_ctx* c, float two_sigA_sqr, float med_scene_depth_lines, float min_affinity, int* out_i, int* out_j,
                              float* out_w, long long cap_edges, long long* out_local2global, long long cap_ids, long long* num_ids)
{
    if (!c) return L3D_ERR_INVALID;
    AffinityState& A = c->aff;
    if (!(min_affinity >= 0.0f)) { c->drop(Stage::Affinity); return l3d_fail(c, L3D_ERR_INVALID, "l3d_affinity_matrix: min_affinity must be >= 0"); }
    const bool cached = A.valid && A.two_sigA_sqr == two_sigA_sqr && A.med == med_scene_depth_lines && A.min_aff == min_affinity;
    if (!cached) c->drop(Stage::Affinity);
    if (!num_ids) return L3D_ERR_INVALID;
    if (!c->sweep.valid) return l3d_fail(c, L3D_ERR_STATE, "l3d_affinity_matrix: call l3d_score_sweep first");
    cudaSetDevice(c->device);
    cudaStream_t st = c->stream;
    if (!cached) {
        const long long ne = affinity_candidates(c, two_sigA_sqr, med_scene_depth_lines, min_affinity);
        if (ne < 0) return ne;
        A.K = 0; A.n_ids = 0;
        if (ne > 0) {
            if (ne >= (1ll << 32) || c->total_segs >= (1ll << 32)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_affinity_matrix: more than 2^32 candidates / segments");
            int rc;
            if ((rc = unused_fixpoint(c, ne)) || (rc = local_ids(c, ne)) || (rc = emit_edges(c, ne))) return rc;
            L3D_CUDA(c, cudaGetLastError(), "affinity matrix kernels");
        }
        A.valid = true; A.two_sigA_sqr = two_sigA_sqr; A.med = med_scene_depth_lines; A.min_aff = min_affinity;
    }
    *num_ids = A.n_ids;
    const long long nE = 2 * A.K;
    if (nE == 0 || !out_i || nE > cap_edges || A.n_ids > cap_ids) return nE;
    L3D_CUDA(c, cudaMemcpyAsync(out_i, A.d_ei.p, 4 * (size_t)nE, cudaMemcpyDeviceToHost, st), "download A");
    L3D_CUDA(c, cudaMemcpyAsync(out_j, A.d_ej.p, 4 * (size_t)nE, cudaMemcpyDeviceToHost, st), "download A");
    L3D_CUDA(c, cudaMemcpyAsync(out_w, A.d_ew.p, 4 * (size_t)nE, cudaMemcpyDeviceToHost, st), "download A");
    if (out_local2global) L3D_CUDA(c, cudaMemcpyAsync(out_local2global, A.d_l2g.p, 8 * (size_t)A.n_ids, cudaMemcpyDeviceToHost, st), "download ids");
    L3D_CUDA(c, cudaStreamSynchronize(st), "affinity matrix download");
    return nE;
}

// replicator_dynamics_diffusion_GPU (cudawrapper.h:80) on a COO edge list (the CLEdge list A_ of line3D.cc:2030).
// out_*: row-sorted COO of the diffused matrix, nnz entries (same order as the reference's downloaded W).
// kernel_ms (optional): device time of the `iters` diffusion iterations only (CUDA events on the context's stream).
// min(w12, w21) of performRDD (line3D.cc:2039-2071): every entry takes the smaller of itself and its transposed entry
__global__ void __launch_bounds__(256) k_rdd_symmetrise(long long nnz, const float* __restrict__ P, const int* __restrict__ tslot, float* __restrict__ out)
{
    const long long y = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= nnz) return;
    const int t = tslot[y];
    out[y] = t >= 0 ? fminf(P[y], P[t]) : P[y];
}

// the diffusion proper on DEVICE edge arrays d_ei/d_ej/d_ew; symmetrise: performRDD's min(w12, w21) applied to the result.  Sets the
// dev of res[0], res[1], res[2] to the result's weights, rows and columns, in row-sorted (i, j) order - the order std::map iterates in
// (line3D.cc:2063-2071); the caller downloads them.  timing (optional): two events, recorded around the `iters` diffusion iterations.
static int rdd_core(l3d_ctx* c, int n, long long nnz, const int* d_ei, const int* d_ej, const float* d_ew, int iters, bool symmetrise,
                    HostBlock res[3], ScopedEvent* timing)
{
    RddState& R = c->rdd;
    int rc;
    L3D_RESERVE(R.d_krow, 8 * nnz, "rdd keys"); L3D_RESERVE(R.d_kcol, 8 * nnz, "rdd keys"); L3D_RESERVE(R.d_k2, 8 * nnz, "rdd keys");
    L3D_RESERVE(R.d_idx, 4 * nnz, "rdd idx"); L3D_RESERVE(R.d_idx2, 4 * nnz, "rdd idx");
    L3D_RESERVE(R.d_P, 4 * nnz, "rdd P"); L3D_RESERVE(R.d_Pn, 4 * nnz, "rdd P'"); L3D_RESERVE(R.d_W, 4 * nnz, "rdd W");
    L3D_RESERVE(R.d_prow, 4 * nnz, "rdd rows"); L3D_RESERVE(R.d_pcol, 4 * nnz, "rdd cols"); L3D_RESERVE(R.d_wmaj, 4 * nnz, "rdd cols"); L3D_RESERVE(R.d_wmin, 4 * nnz, "rdd rows");
    L3D_RESERVE(R.d_rowptr, 4 * ((long long)n + 1), "rdd rowptr"); L3D_RESERVE(R.d_colptr, 4 * ((long long)n + 1), "rdd colptr"); L3D_RESERVE(R.d_tslot, 4 * nnz, "rdd tslot");
    cudaStream_t st = c->stream;
    const unsigned int nb = (unsigned int)((nnz + 255) / 256);
    k_rdd_keys<<<nb, 256, 0, st>>>(nnz, d_ei, d_ej, (unsigned long long*)R.d_krow.p, (unsigned long long*)R.d_kcol.p, (unsigned int*)R.d_idx.p);
    // P: row-sorted (stable, like std::list::sort with sortCLEdgesByRow, sparsematrix.cc:22-25 / 104-107), W: col-sorted
    auto sort_by = [&](const DevBuf& keys) {
        return l3d_cub(c, "rdd sort", [&](void* tmp, size_t& bytes) {
            return cub::DeviceRadixSort::SortPairs(tmp, bytes, (const unsigned long long*)keys.p, (unsigned long long*)R.d_k2.p, (const unsigned int*)R.d_idx.p,
                                                   (unsigned int*)R.d_idx2.p, (int)nnz, 0, 64, st); });
    };
    if ((rc = sort_by(R.d_krow))) return rc;
    k_rdd_gather<<<nb, 256, 0, st>>>(nnz, (const unsigned long long*)R.d_k2.p, (const unsigned int*)R.d_idx2.p, d_ew, (float*)R.d_P.p, (int*)R.d_prow.p, (int*)R.d_pcol.p);
    if ((rc = sort_by(R.d_kcol))) return rc;
    k_rdd_gather<<<nb, 256, 0, st>>>(nnz, (const unsigned long long*)R.d_k2.p, (const unsigned int*)R.d_idx2.p, d_ew, (float*)R.d_W.p, (int*)R.d_wmaj.p, (int*)R.d_wmin.p);
    k_rdd_ptr<<<(n + 256) / 256, 256, 0, st>>>(n, (int)nnz, (const int*)R.d_prow.p, (int*)R.d_rowptr.p);
    k_rdd_ptr<<<(n + 256) / 256, 256, 0, st>>>(n, (int)nnz, (const int*)R.d_wmaj.p, (int*)R.d_colptr.p);
    k_rdd_tslot<<<nb, 256, 0, st>>>(nnz, (const int*)R.d_prow.p, (const int*)R.d_pcol.p, (const int*)R.d_rowptr.p, (int*)R.d_tslot.p);
    // padded value arrays (rows / columns on float4 boundaries)
    L3D_RESERVE(R.d_len4, 4 * ((long long)n + 1), "rdd len4"); L3D_RESERVE(R.d_rp4, 4 * ((long long)n + 1), "rdd rp4"); L3D_RESERVE(R.d_cp4, 4 * ((long long)n + 1), "rdd cp4");
    int tot4[2] = {0, 0};
    for (int pass = 0; pass < 2; ++pass) {
        const int* ptr = (const int*)(pass ? R.d_colptr.p : R.d_rowptr.p);
        int* p4 = (int*)(pass ? R.d_cp4.p : R.d_rp4.p);
        L3D_CUDA(c, cudaMemsetAsync(R.d_len4.p, 0, 4 * ((size_t)n + 1), st), "rdd len4");
        k_rdd_len4<<<(n + 255) / 256, 256, 0, st>>>(n, ptr, (int*)R.d_len4.p);
        if ((rc = l3d_cub(c, "rdd scan", [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, (const int*)R.d_len4.p, p4, n + 1, st); }))) return rc;
        L3D_CUDA(c, cudaMemcpyAsync(&tot4[pass], p4 + n, 4, cudaMemcpyDeviceToHost, st), "rdd padded size");
    }
    L3D_CUDA(c, cudaStreamSynchronize(st), "rdd padded size");
    const size_t pbytes = 16 * (size_t)std::max(tot4[0], 1), wbytes = 16 * (size_t)std::max(tot4[1], 1);
    L3D_RESERVE(R.d_Pp, pbytes, "rdd P padded"); L3D_RESERVE(R.d_Pnp, pbytes, "rdd P' padded"); L3D_RESERVE(R.d_Wp, wbytes, "rdd W padded");
    L3D_CUDA(c, cudaMemsetAsync(R.d_Pp.p, 0, pbytes, st), "rdd pad"); L3D_CUDA(c, cudaMemsetAsync(R.d_Wp.p, 0, wbytes, st), "rdd pad");
    k_rdd_pad<<<nb, 256, 0, st>>>(nnz, (const int*)R.d_prow.p, (const int*)R.d_rowptr.p, (const int*)R.d_rp4.p, (const float*)R.d_P.p, (float*)R.d_Pp.p);
    k_rdd_pad<<<nb, 256, 0, st>>>(nnz, (const int*)R.d_wmaj.p, (const int*)R.d_colptr.p, (const int*)R.d_cp4.p, (const float*)R.d_W.p, (float*)R.d_Wp.p);
    if (4ll * std::max(tot4[0], tot4[1]) >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_rdd: padded matrix too large for 32-bit slots");
    L3D_RESERVE(R.d_plan, 16 * nnz, "rdd plan"); L3D_RESERVE(R.d_dst, 4 * nnz, "rdd dst");
    k_rdd_plan<<<nb, 256, 0, st>>>(nnz, (const int*)R.d_prow.p, (const int*)R.d_pcol.p, (const int*)R.d_rowptr.p, (const int*)R.d_colptr.p,
                                   (const int*)R.d_rp4.p, (const int*)R.d_cp4.p, (const int*)R.d_tslot.p, (int4*)R.d_plan.p, (int*)R.d_dst.p);
    // P' starts as a copy of the un-normalised P (cudawrapper.cu:724), then P is row-normalised (727)
    L3D_CUDA(c, cudaMemcpyAsync(R.d_Pnp.p, R.d_Pp.p, pbytes, cudaMemcpyDeviceToDevice, st), "rdd copy");
    const unsigned int nbn = (unsigned int)((4ll * n + 255) / 256);
    auto normalize = [&](float* Pbuf) { k_rdd_normalize_q<<<nbn, 256, 0, st>>>(n, (const int*)R.d_rowptr.p, (const int*)R.d_rp4.p, Pbuf); };
    normalize((float*)R.d_Pp.p);
    if (timing) {
        if ((rc = timing[0].create(c)) || (rc = timing[1].create(c))) return rc;
        cudaEventRecord(timing[0].e, st);
    }
    float* P = (float*)R.d_Pp.p; float* Pn = (float*)R.d_Pnp.p;
    for (int it = 0; it < iters; ++it) {
        k_rdd_step8<<<(unsigned int)((nnz + 255) / 256), 256, 0, st>>>(nnz, (const int4*)R.d_plan.p, (const int*)R.d_dst.p, P, (const float*)R.d_Wp.p, Pn);
        std::swap(P, Pn);
        if (it < iters - 1) normalize(P);       // no normalisation after the last step (cudawrapper.cu:751)
    }
    if (timing) cudaEventRecord(timing[1].e, st);
    k_rdd_unpad<<<nb, 256, 0, st>>>(nnz, (const int*)R.d_prow.p, (const int*)R.d_rowptr.p, (const int*)R.d_rp4.p, P, (float*)R.d_P.p);
    res[0].dev = R.d_P.p;
    if (symmetrise) {
        k_rdd_symmetrise<<<nb, 256, 0, st>>>(nnz, (const float*)R.d_P.p, (const int*)R.d_tslot.p, (float*)R.d_Pn.p);
        res[0].dev = R.d_Pn.p;
        ++c->launches;
    }
    c->launches += 9 + 16 + 10 + 2 * iters;
    L3D_CUDA(c, cudaGetLastError(), "rdd kernels");
    res[1].dev = R.d_prow.p; res[2].dev = R.d_pcol.p;
    return L3D_OK;
}

int l3d_rdd(l3d_ctx* c, int n, long long nnz, const int* ei, const int* ej, const float* ew, int iters, int* out_i, int* out_j,
            float* out_w, float* kernel_ms)
{
    if (!c || n <= 0 || nnz < 0 || (nnz && (!ei || !ej || !ew || !out_i || !out_j || !out_w))) return l3d_fail(c, L3D_ERR_INVALID, "l3d_rdd: bad arguments");
    if (nnz == 0) return L3D_OK;
    if (nnz >= (1ll << 31) - 2) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_rdd: more than 2^31 entries");
    cudaSetDevice(c->device);
    int rc;
    HostBlock in[3] = {host_array(ei, 4 * nnz), host_array(ej, 4 * nnz), host_array(ew, 4 * nnz)};
    HostBlock res[3] = {host_array(out_w, 4 * nnz), host_array(out_i, 4 * nnz), host_array(out_j, 4 * nnz)};
    ScopedEvent timing[2];
    if ((rc = l3d_stage_host(c, in, 3, nullptr, 0)) ||
        (rc = rdd_core(c, n, nnz, (const int*)in[0].dev, (const int*)in[1].dev, (const float*)in[2].dev, iters, false, res, kernel_ms ? timing : nullptr)) ||
        (rc = l3d_unstage_host(c, res, 3, "rdd")))
        return rc;
    if (kernel_ms) cudaEventElapsedTime(kernel_ms, timing[0].e, timing[1].e);
    return L3D_OK;
}

// performRDD (line3D.cc:2026-2076) on the affinity matrix l3d_affinity_matrix left on the device: no download / re-upload of A_, the
// min(w12, w21) symmetrisation on the device, the result in the (i, j) order the reference rebuilds A_ in.  out arrays: 2 * K entries
// (the count l3d_affinity_matrix returned).
long long l3d_rdd_affinity(l3d_ctx* c, int iters, int* out_i, int* out_j, float* out_w, long long cap)
{
    if (!c || !out_i || !out_j || !out_w) return L3D_ERR_INVALID;
    AffinityState& A = c->aff;
    if (!A.valid) return l3d_fail(c, L3D_ERR_STATE, "l3d_rdd_affinity: call l3d_affinity_matrix first");
    const long long nnz = 2 * A.K;
    if (nnz == 0 || nnz > cap) return nnz;
    if (nnz >= (1ll << 31) - 2) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_rdd_affinity: more than 2^31 entries");
    cudaSetDevice(c->device);
    int rc;
    HostBlock res[3] = {host_array(out_w, 4 * nnz), host_array(out_i, 4 * nnz), host_array(out_j, 4 * nnz)};
    if ((rc = rdd_core(c, (int)A.n_ids, nnz, (const int*)A.d_ei.p, (const int*)A.d_ej.p, (const float*)A.d_ew.p, iters, true, res, nullptr))) return rc;
    return (rc = l3d_unstage_host(c, res, 3, "rdd")) ? rc : nnz;
}

// Stable ascending argsort of float keys on the device (the edge-weight sort of performClustering, clustering.cc:13-14:
// std::list::sort by weight is stable).  perm_out[i] = index of the i-th smallest key; equal keys keep their input order.
int l3d_argsort_f32(l3d_ctx* c, long long n, const float* keys, unsigned int* perm_out)
{
    if (!c || n < 0 || (n && (!keys || !perm_out))) return l3d_fail(c, L3D_ERR_INVALID, "l3d_argsort_f32: bad arguments");
    if (n == 0) return L3D_OK;
    if (n >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_argsort_f32: more than 2^31 keys");
    cudaSetDevice(c->device);
    RddState& R = c->rdd;
    int rc;
    L3D_RESERVE(R.d_k2, 4 * n, "sort keys"); L3D_RESERVE(R.d_idx, 4 * n, "sort idx");
    HostBlock in[1] = {host_array(keys, 4 * (size_t)n)}, out[1] = {host_array(perm_out, 4 * (size_t)n)};
    if ((rc = l3d_stage_host(c, in, 1, out, 1))) return rc;
    cudaStream_t st = c->stream;
    k_iota<<<(unsigned int)((n + 255) / 256), 256, 0, st>>>(n, (unsigned int*)R.d_idx.p);
    if ((rc = l3d_cub(c, "argsort", [&](void* tmp, size_t& bytes) {
             return cub::DeviceRadixSort::SortPairs(tmp, bytes, (const float*)in[0].dev, (float*)R.d_k2.p, (const unsigned int*)R.d_idx.p, (unsigned int*)out[0].dev, (int)n, 0, 32, st); })))
        return rc;
    c->launches += 6;
    return l3d_unstage_host(c, out, 1, "argsort");
}

} // extern "C"
