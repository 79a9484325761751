// l3d_device.cuh — device-side types and the selection-critical arithmetic of the matching path.
//
// ARITHMETIC CONTRACT.  This translation unit is compiled with -fmad=false: every `a*b + c` written in plain C++ is
// two IEEE-754 roundings.  The functions in the "exact" section perform, operation for operation, the float
// arithmetic of the reference kernels (cudawrapper.cu:18-164 with helper_math.h:1248/1291/1309/1420) so that
// `overlap`, the four depths and therefore kNN membership are BIT-IDENTICAL to the reference built with
// nvcc -fmad=false (oracle/_ref/libl3dref_nofma.so).  Anything that is allowed to be approximate (the conservative
// pre-filter) spells its fused multiply-adds explicitly with __fmaf_rn and never decides a result on its own:
// it only proves "this pair cannot survive" with a safety margin, everything else goes through the exact path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define L3D_EPS_F 1e-12f   /* __device__ const float L3D_EPS_GPU = 1e-12  (cudawrapper.h:50) */

// ---- device-resident descriptors --------------------------------------------------------------------------------
struct L3DViewDev {
    long long seg_off;      // first segment of this view in the flat float4 segment array
    int nseg;
    unsigned int cam_id;
    int width, height;
    float RtKinv[9];        // float R^T K^-1 (view.cc:37-40)
    float C[3];             // float camera centre, untranslated (view.cc:35)
    float k, median_depth;
    double RtKinv_d[9];
    double C_d[3];
};

struct L3DPairDev {
    int src, tgt;           // view indices
    float F[9];             // row-major float fundamental matrix
    long long row_off;      // first output row of this pair (prefix sum of Ns)
    double Fd[9];           // the double matrix (REF_CPU semantics, l3d_match_pairs_f64); unused otherwise
    long long arc_off;      // first entry of this pair in the array of target arcs (level-1 pre-filter, k_pair_arcs)
};

// "which entry owns index x" over a table of first indices: the last i in [0, n) with key(i) <= x, 0 if there is none.
// key(i) must not decrease with i; n >= 1.
template <typename T, typename Key>
__device__ __forceinline__ int last_le(int n, T x, Key key)
{
    int lo = 0, hi = n - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (key(mid) <= x) lo = mid; else hi = mid - 1; }
    return lo;
}

// ---- level-1 pre-filter: the pencil parameter -----------------------------------------------------------------------
// All epipolar lines F*p of one view pair pass through the epipole E of the target image, i.e. they live in the 2-D subspace
// {e : e . E = 0} of R^3.  With image coordinates divided by L3D_ARC_SCALE (so that points are ~unit vectors and the subspace is
// well conditioned whether E lies inside the image or at infinity) and (u, v) an orthonormal basis of that subspace, the angle
//     kappa(e) = atan2(e.v, e.u)   (mod pi)
// is a 1-D coordinate of the pencil; the pencil line through an image point x has kappa(x) = atan2(x.u, -x.v).  Along a target
// line l the map kappa -> intersection point is monotone on the circle cut at kappa_l (the pencil line parallel to l), so a target
// segment [q1, q2] is an ARC T of the circle, and so is the stretch T_ext of its line between t = -X and t = 1 + X (t = 0 at q1,
// 1 at q2, X = 1/epi_overlap + 0.5).  The reference's overlap (cudawrapper.cu:89-136) is inner / outer length of two collinear
// intervals, hence
//   * 0 when the projections of both epipolar lines of a source segment fall outside [q1, q2] on the SAME side (both kappa below T
//     or both above T),
//   * below epi_overlap when either projection is farther than X segment lengths away (outer > X, inner <= 1): a kappa outside T_ext.
// A row can therefore only match targets with both kappa inside T_ext and not on the same side of T - which implies that T meets the
// short arc [ka, kb] between the two kappa values, i.e. that T starts in [ka - |T|, kb].  The targets of a view pair are therefore grouped
// into L3D_ARC_NCLS classes by the length of T (class c: |T| <= 2^(L3D_ARC_CLS0 + c)) and sorted by the start of T inside a class: a
// row's candidates are one WINDOW [ka - 2^(L3D_ARC_CLS0 + c), kb] per class (k_match_topk); targets without a usable arc form a last
// class that every row looks at.  Angles are stored in units of pi / 2^32: unsigned subtraction wraps mod pi for free.
#define L3D_ARC_SCALE 2048.0
#define L3D_ARC_NCLS 8
#define L3D_ARC_CLS0 21
struct L3DPairBasis { double u[3], v[3]; int cls_off[L3D_ARC_NCLS + 2]; };    // + first sorted entry of every class of the pair, and the end
__device__ __forceinline__ int arc_class(unsigned int len)      // L3D_ARC_NCLS = no usable arc / longer than the last class
{
    if (len == 0xFFFFFFFFu) return L3D_ARC_NCLS;
    const int b = len <= 1u ? 0 : 32 - __clz(len - 1u);          // ceil(log2(len))
    return b <= L3D_ARC_CLS0 ? 0 : min(b - L3D_ARC_CLS0, L3D_ARC_NCLS);
}
#define L3D_ARC_WIDE 0x80000000u      /* entry.z flag: no usable arc (epipole too close, degenerate segment, arc too long): always a candidate */
// sorted entry: x = start A of T (absolute), y = e1 | w << 16, z = ehi | flag, w = target index; e1 / w / ehi = length of T_ext below T,
// of T, of T_ext above T in units of 2^16 (rounded up).  Both kappa inside T_ext, not both below T, not both above T.
__device__ __forceinline__ bool arc_may_match(uint4 e, unsigned int k1, unsigned int k2)
{
    const unsigned int E1 = e.y << 16, E2 = E1 + (e.y & 0xFFFF0000u), E3 = E2 + (e.z << 16);
    const unsigned int base = e.x - E1, d1 = k1 - base, d2 = k2 - base, mx = max(d1, d2), mn = min(d1, d2);
    return (mx <= E3 && mx >= E1 && mn <= E2) || (e.z & L3D_ARC_WIDE);
}
__device__ __forceinline__ unsigned int arc_units(double kappa)
{ return (unsigned int)(long long)llrint(kappa * (4294967296.0 / 3.14159265358979323846)); }
// kappa of an epipolar line (float, exactly as the kernels form it).  *off: the line misses the pencil by more than 0.02 px inside
// the image (its component along n = u x v, i.e. a source point so close to the epipole that F*p is rounding noise): the 1-D model
// does not describe it and the row must skip level 1.
__device__ __forceinline__ unsigned int line_kappa(const L3DPairBasis& B, float3 e, bool* off)
{
    const double x = L3D_ARC_SCALE * (double)e.x, y = L3D_ARC_SCALE * (double)e.y, z = (double)e.z;
    const double cu = x * B.u[0] + y * B.u[1] + z * B.u[2], cv = x * B.v[0] + y * B.v[1] + z * B.v[2];
    const double nx = B.u[1] * B.v[2] - B.u[2] * B.v[1], ny = B.u[2] * B.v[0] - B.u[0] * B.v[2], nz = B.u[0] * B.v[1] - B.u[1] * B.v[0];
    const double cn = x * nx + y * ny + z * nz, exy = sqrt((double)e.x * (double)e.x + (double)e.y * (double)e.y);
    const double k = atan2(cv, cu);
    *off = !(4.0 * fabs(cn) <= 0.02 * exy) || !isfinite(k);     // |n . x| <= ~3 for scaled image points
    return isfinite(k) ? arc_units(k) : 0u;
}

// per-segment cache written by k_prep_segments: 3 float4 per segment
//   c0 = (ray1.x, ray1.y, ray1.z, ray2.x)  c1 = (ray2.y, ray2.z, n.x, n.y)  c2 = (n.z, 0, 0, 0)
struct SegRays { float3 r1, r2, n; };

__device__ __forceinline__ SegRays load_rays(const float4* __restrict__ cache, long long idx)
{
    float4 a = __ldg(cache + 3 * idx), b = __ldg(cache + 3 * idx + 1), c = __ldg(cache + 3 * idx + 2);
    SegRays s;
    s.r1 = make_float3(a.x, a.y, a.z);
    s.r2 = make_float3(a.w, b.x, b.y);
    s.n = make_float3(b.z, b.w, c.x);
    return s;
}
// the same three float4 from shared memory
__device__ __forceinline__ SegRays rays_from_smem(const float4* p)
{
    const float4 a = p[0], b = p[1], c = p[2];
    SegRays s;
    s.r1 = make_float3(a.x, a.y, a.z); s.r2 = make_float3(a.w, b.x, b.y); s.n = make_float3(b.z, b.w, c.x);
    return s;
}

// =============================================================================== exact section (reference op order)
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 cross3(float3 a, float3 b)
{ return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float3 normalize3(float3 v)
{ float inv = rsqrtf(dot3(v, v)); return make_float3(v.x * inv, v.y * inv, v.z * inv); }
// 3x3 row-major matrix times (x, y, 1): ((0 + m0*x) + m1*y) + m2*1   (cudawrapper.cu:56-75)
__device__ __forceinline__ float3 mulmat_h(const float* __restrict__ m, float x, float y)
{
    float3 o;
    o.x = 0.0f; o.x += m[0] * x; o.x += m[1] * y; o.x += m[2] * 1.0f;
    o.y = 0.0f; o.y += m[3] * x; o.y += m[4] * y; o.y += m[5] * 1.0f;
    o.z = 0.0f; o.z += m[6] * x; o.z += m[7] * y; o.z += m[8] * 1.0f;
    return o;
}
// dot((p1-q),(p2-q)) < eps on the xy parts  (cudawrapper.cu:80-86)
__device__ __forceinline__ bool on_seg(float p1x, float p1y, float p2x, float p2y, float qx, float qy)
{
    float v1x = p1x - qx, v1y = p1y - qy, v2x = p2x - qx, v2y = p2y - qy;
    return (v1x * v2x + v1y * v2y) < L3D_EPS_F;
}
__device__ __forceinline__ float len2d(float ax, float ay, float bx, float by)
{
    float dx = ax - bx, dy = ay - by;
    return sqrtf(dx * dx + dy * dy);   // length(float3) with z difference 0 (helper_math.h:1291)
}

// Epipolar overlap of tgt segment q=(x1,y1,x2,y2) with the epipolar beam (e1,e2) of a src segment.
// Follows K_match_lines cudawrapper.cu:213-232 + D_segment_overlap_2D 89-136.  *invalid is set when an
// intersection is degenerate (cudawrapper.cu:223-229): the reference then reports overlap 0 and depths -1.
__device__ __forceinline__ float exact_overlap(float4 q, float3 e1, float3 e2, bool* invalid)
{
    *invalid = false;
    // l_tgt = cross((x1,y1,1),(x2,y2,1))
    float3 l = make_float3(q.y * 1.0f - 1.0f * q.w, 1.0f * q.z - q.x * 1.0f, q.x * q.w - q.y * q.z);
    float3 a = cross3(l, e1), b = cross3(l, e2);
    if (!(fabsf(a.z) > L3D_EPS_F) || !(fabsf(b.z) > L3D_EPS_F)) { *invalid = true; return 0.0f; }
    float ax = a.x / a.z, ay = a.y / a.z, bx = b.x / b.z, by = b.y / b.z;   // projected endpoints on the tgt line
    float len_src = len2d(q.x, q.y, q.z, q.w);
    float len_tgt = len2d(ax, ay, bx, by);
    if (len_src < 1.0f || len_tgt < 1.0f) return 0.0f;
    bool A = on_seg(q.x, q.y, q.z, q.w, ax, ay);   // proj1 inside tgt segment
    bool B = on_seg(q.x, q.y, q.z, q.w, bx, by);   // proj2 inside tgt segment
    bool Cc = on_seg(ax, ay, bx, by, q.x, q.y);    // tgt p1 inside projected interval
    bool D = on_seg(ax, ay, bx, by, q.z, q.w);     // tgt p2 inside projected interval
    // The reference's case analysis (cudawrapper.cu:99-131) returns a ratio of two lengths in every case.  Written without branches -
    // operands selected first, then the same sqrtf / division on the same values - so that the 32 candidates of a batch do not
    // serialise over five different paths:
    //   A && B        : len_tgt / len_src                    Cc && D       : len_src / len_tgt
    //   A (b outside) : len1 = |q2 - b|, len2 = |q1 - b|;    Cc && len1 > 1 ? |a - q1| / len1 : len2 > 1 ? |a - q2| / len2 : 0
    //   B (a outside) : len1 = |q1 - a|, len2 = |q2 - a|;    D  && len1 > 1 ? |b - q2| / len1 : len2 > 1 ? |b - q1| / len2 : 0
    const bool cAB = A && B, cCD = !cAB && Cc && D, cA = !cAB && !cCD && A, cB = !cAB && !cCD && !A && B;
    const float fx = cA ? bx : ax, fy = cA ? by : ay;            // the projection outside the tgt segment
    const float ix = cA ? ax : bx, iy = cA ? ay : by;            // the projection inside it
    const float u1x = cA ? q.z : q.x, u1y = cA ? q.w : q.y;      // tgt end point of len1
    const float u2x = cA ? q.x : q.z, u2y = cA ? q.y : q.w;      // tgt end point of len2
    const float len1 = len2d(u1x, u1y, fx, fy), len2 = len2d(u2x, u2y, fx, fy);
    const bool first = (cA ? Cc : D) && len1 > 1.0f, second = !first && len2 > 1.0f;
    const float num1 = len2d(ix, iy, first ? u2x : u1x, first ? u2y : u1y);
    const float num = cAB ? len_tgt : cCD ? len_src : num1;
    const float den = cAB ? len_src : cCD ? len_tgt : first ? len1 : len2;
    const bool any = cAB || cCD || ((cA || cB) && (first || second));
    const float r = num / den;
    return any ? r : 0.0f;
}

// numerator of the depths on the plane through camera centre Ca with normal n, seen from camera centre Cb
__device__ __forceinline__ float depth_num(float3 n, float3 Ca, float3 Cb) { return dot3(Ca, n) - dot3(n, Cb); }

// The two D_triangulate_depth calls of K_match_lines (cudawrapper.cu:139-164, 237-242) from cached rays / normals.
//   d[0],d[1]: depths of the src endpoints on the plane (C_tgt, tgt segment)
//   d[2],d[3]: depths of the tgt endpoints on the plane (C_src, src segment)
__device__ __forceinline__ void exact_depths(const SegRays& s, const SegRays& t, float3 Cs, float3 Ct, float* d)
{
    d[0] = d[1] = d[2] = d[3] = -1.0f;
    {
        float dp1 = dot3(t.n, s.r1), dp2 = dot3(t.n, s.r2);
        if (!(fabsf(dp1) < L3D_EPS_F || fabsf(dp2) < L3D_EPS_F)) {
            float num = depth_num(t.n, Ct, Cs);
            d[0] = num / dp1; d[1] = num / dp2;
        }
    }
    {
        float dq1 = dot3(s.n, t.r1), dq2 = dot3(s.n, t.r2);
        if (!(fabsf(dq1) < L3D_EPS_F || fabsf(dq2) < L3D_EPS_F)) {
            float num = depth_num(s.n, Cs, Ct);
            d[2] = num / dq1; d[3] = num / dq2;
        }
    }
}

// True exactly when exact_depths(s, t, Cs, Ct, d) makes all four d > 0, without its four divisions; num_s = depth_num(s.n, Cs, Ct).
// Each depth is num / dp with |dp| >= L3D_EPS_F (else -1), and |dp| <= 1 + 1e-6: both factors are unit vectors normalised with
// rsqrtf, or NaN.  Denormals are kept (no -ftz), so a finite num != 0 gives a quotient of magnitude at least 2^-149 / (1 + 1e-6)
// before rounding, above the 2^-150 midpoint: it never rounds to 0, and num / dp > 0 exactly when num and dp are nonzero with the
// same sign.  NaN fails both forms; an infinite quotient passes both when the signs agree.
__device__ __forceinline__ bool same_sign(float a, float b) { return (a > 0.0f && b > 0.0f) || (a < 0.0f && b < 0.0f); }
__device__ __forceinline__ bool depths_in_front(const SegRays& s, const SegRays& t, float3 Cs, float3 Ct, float num_s)
{
    const float dp1 = dot3(t.n, s.r1), dp2 = dot3(t.n, s.r2), dq1 = dot3(s.n, t.r1), dq2 = dot3(s.n, t.r2);
    if (fabsf(dp1) < L3D_EPS_F || fabsf(dp2) < L3D_EPS_F || fabsf(dq1) < L3D_EPS_F || fabsf(dq2) < L3D_EPS_F) return false;
    const float num_t = depth_num(t.n, Ct, Cs);
    return same_sign(num_t, dp1) && same_sign(num_t, dp2) && same_sign(num_s, dq1) && same_sign(num_s, dq2);
}

// =============================================================================== conservative pre-filter
// Row constants for the filter: epipolar lines e1,e2 of the src endpoints and g = c1 * max(|e1.xy|, |e2.xy|).
// Parametrise the tgt line by t (t=0 at q1, t=1 at q2).  The epipolar line e_i meets it at
//     t_i = a_i / (a_i - b_i),  a_i = e_i . (q1,1),  b_i = e_i . (q2,1),
// so the projected interval is [min t, max t] and the reference's overlap score equals
//     (min(1,tmax) - max(0,tmin)) / (max(1,tmax) - min(0,tmin))      (inner / outer length of two collinear intervals).
// The reference evaluates this through 2-D intersections in float; its rounding error, expressed in t, is bounded by
// ~2.4e-4 * |e.xy| / |a-b| (cancellation in l.z ~ 4000*|d|) plus a relative 6e-8/sin(phi) on |t|.  The filter rejects a
// pair only if, with margin m = m0 + g/|a-b| on both interval ends and 5 % slack on the threshold, the score cannot
// exceed `thr`.  NaN/Inf (a-b == 0, i.e. epipolar line parallel to the segment) never reject.
#define L3D_FILTER_M0 2e-3f
#define L3D_FILTER_C1 4e-3f
__device__ __forceinline__ float rcp_approx(float x)
{ float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }   // MUFU.RCP, 1 ulp; the filter has 1e-3 margins
// rA = (e1.x, e1.y, e1.z, e2.x)  rB = (e2.y, e2.z, g, thr_scaled)   thr_scaled = 0.95 * (score a pair must exceed)
__device__ __forceinline__ bool filter_may_survive(float4 q, float4 rA, float4 rB)
{
    float a1 = __fmaf_rn(rA.x, q.x, __fmaf_rn(rA.y, q.y, rA.z));
    float b1 = __fmaf_rn(rA.x, q.z, __fmaf_rn(rA.y, q.w, rA.z));
    float a2 = __fmaf_rn(rA.w, q.x, __fmaf_rn(rB.x, q.y, rB.y));
    float b2 = __fmaf_rn(rA.w, q.z, __fmaf_rn(rB.x, q.w, rB.y));
    float r1 = rcp_approx(a1 - b1), r2 = rcp_approx(a2 - b2);
    float t1 = a1 * r1, t2 = a2 * r2;
    float tmin = fminf(t1, t2), tmax = fmaxf(t1, t2);
    float inner = fminf(tmax, 1.0f) - fmaxf(tmin, 0.0f);
    float outer = fmaxf(tmax, 1.0f) - fminf(tmin, 0.0f);
    float m = __fmaf_rn(rB.z, fmaxf(fabsf(r1), fabsf(r2)), L3D_FILTER_M0);
    // survive  <=>  inner + 2m > thr_scaled * (outer - 2m)   <=>  inner - thr_scaled*outer + (2 + 2*thr_scaled)*m > 0
    float v = __fmaf_rn(__fmaf_rn(2.0f, rB.w, 2.0f), m, __fmaf_rn(-rB.w, outer, inner));
    // The reference's case analysis (which endpoint lies inside which interval, cudawrapper.cu:99-131) is decided by
    // the signs of t and t-1.  If an intersection sits within m of a segment end, its float evaluation may take a
    // different branch than the geometry suggests (and then return a ratio unrelated to inner/outer), so such pairs
    // are never rejected here.  dist_i = | |t_i - 1/2| - 1/2 | = distance of t_i to the nearer of {0, 1}.
    float dist = fminf(fabsf(fabsf(t1 - 0.5f) - 0.5f), fabsf(fabsf(t2 - 0.5f) - 0.5f));
    return !(v <= 0.0f) || !(dist > m);   // NaN -> true
}

// 64-bit selection key: larger overlap first, ties broken by the smaller tgt index (overlap > 0 so its bit pattern
// is monotone as an unsigned integer).
__device__ __forceinline__ unsigned long long make_key(float overlap, unsigned int tgt)
{ return ((unsigned long long)__float_as_uint(overlap) << 32) | (unsigned long long)(0xFFFFFFFFu - tgt); }
__device__ __forceinline__ float key_overlap(unsigned long long k) { return __uint_as_float((unsigned int)(k >> 32)); }
__device__ __forceinline__ unsigned int key_tgt(unsigned long long k) { return 0xFFFFFFFFu - (unsigned int)(k & 0xFFFFFFFFull); }

// ---- mbarrier + 1-D TMA (cp.async.bulk) ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned int count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned int bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned int parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// bulk async copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, unsigned int bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
