// l3d_device_f64.cuh — double-precision device arithmetic: the host-side double code of view.cc / line3D.cc and the
// reference's CPU twins (matchingCPU line3D.cc:900-1015, scoringCPU 1208-1294) restated for the device.
// This is the single home of the device's double geometry: the 3-vector and its operations, Segment3D and the
// undirected angle between 3D segments.  Every kernel that needs one of them includes this header instead of
// restating it, so a parity fix lands in one place.
//
// ARITHMETIC CONTRACT.  Compiled with -fmad=false; IEEE double add/mul/div/sqrt on the GPU round exactly like the host's,
// so everything here that uses only those operations is bit-identical to oracle/l3d_oracle.cc (built with
// -ffp-contract=off), which restates the reference's Eigen expressions component by component.
#pragma once
#include "l3d_device.cuh"

#define L3D_EPS_D 1e-12
#define L3D_PI_D 3.14159265358979323846

struct D3 { double x, y, z; };
__device__ __forceinline__ D3 d3(double x, double y, double z) { D3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ D3 dsub(D3 a, D3 b) { return d3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double ddot(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ D3 dcross(D3 a, D3 b) { return d3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ double dnorm(D3 a) { return sqrt(ddot(a, a)); }
__device__ __forceinline__ D3 dnormalized(D3 a)
{
    double n2 = ddot(a, a);
    if (n2 > 0) { double n = sqrt(n2); return d3(a.x / n, a.y / n, a.z / n); }
    return a;
}
__device__ __forceinline__ D3 dmulmat(const double* M, D3 v)
{ return d3(M[0] * v.x + M[1] * v.y + M[2] * v.z, M[3] * v.x + M[4] * v.y + M[5] * v.z, M[6] * v.x + M[7] * v.y + M[8] * v.z); }
// View::getNormalizedRay (view.cc:317-321)
__device__ __forceinline__ D3 dray(const double* M, double x, double y) { return dnormalized(dmulmat(M, d3(x, y, 1.0))); }

// Segment3D(P1, P2) (segment3D.h:48-66): a segment whose float length is not above 1e-12 collapses to zero.
// n2 > 1e-20 already implies (float)sqrt(n2) > 1e-12; testing it first keeps the sqrt off the common path of callers
// that only need the direction.  Selects rather than if/else: the branching form gave the affinity stage's earlier
// per-segment event kernel 102 registers instead of 94, one resident CTA less per SM, and made it 20 % slower.
struct Seg3D { D3 P1, P2, dir; float length; };
__device__ __forceinline__ Seg3D seg3d(D3 P1, D3 P2)
{
    const D3 d = dsub(P1, P2);
    const double n2 = ddot(d, d);
    const float length = (float)sqrt(n2);
    const bool valid = n2 > 1e-20 || length > L3D_EPS_D;
    const D3 zero = d3(0, 0, 0);
    Seg3D s;
    s.P1 = valid ? P1 : zero;
    s.P2 = valid ? P2 : zero;
    s.dir = valid ? dnormalized(dsub(P2, P1)) : zero;
    s.length = valid ? length : 0.0f;
    return s;
}
// Segment3D::distance_Point2Line (segment3D.h:69-73): P1 + (dir * (P-P1)^T) * dir, evaluated as (outer product) * dir
__device__ __forceinline__ float dist_p2l(const Seg3D& s, D3 P)
{
    const D3 w = dsub(P, s.P1);
    const double d[3] = {s.dir.x, s.dir.y, s.dir.z}, ww[3] = {w.x, w.y, w.z};
    double h[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) h[i] = (d[i] * ww[0]) * d[0] + (d[i] * ww[1]) * d[1] + (d[i] * ww[2]) * d[2];
    return (float)dnorm(dsub(d3(s.P1.x + h[0], s.P1.y + h[1], s.P1.z + h[2]), P));
}
// undirected angle in degrees, [0, 90], from the float cosine of two directions: D_undirected_angle_3D_DEG
// (cudawrapper.cu:46-53) and angleBetweenSeg3D (line3D.cc:1571-1583) alike: float acos, DOUBLE divide by pi, times 180, back to float
__device__ __forceinline__ float undirected_angle_deg(float c)
{
    float angle = (float)((double)acosf(fmaxf(fminf(c, 1.0f), -1.0f)) / L3D_PI_D * (double)180.0f);
    if (angle > 90.0f) angle = 180.0f - angle;
    return angle;
}

// ---- matchingCPU -------------------------------------------------------------------------------------------------
// per-segment cache of the double path: viewing rays of both endpoints and the normalised normal of their plane
// (triangulationDepths line3D.cc:1168-1193 recomputes these per surviving pair); 9 doubles per segment
struct SegRaysD { D3 r1, r2, n; };
__device__ __forceinline__ SegRaysD load_rays_d(const double* __restrict__ cache, long long idx)
{
    const double* p = cache + 9 * idx;
    SegRaysD s;
    s.r1 = d3(__ldg(p), __ldg(p + 1), __ldg(p + 2)); s.r2 = d3(__ldg(p + 3), __ldg(p + 4), __ldg(p + 5)); s.n = d3(__ldg(p + 6), __ldg(p + 7), __ldg(p + 8));
    return s;
}
// pointOnSegment (line3D.cc:1077-1083): x between p1 and p2 (2-D)
__device__ __forceinline__ bool d_on_seg(D3 x, D3 p1, D3 p2) { return ((p1.x - x.x) * (p2.x - x.x) + (p1.y - x.y) * (p2.y - x.y)) < L3D_EPS_D; }

// Epipolar overlap of matchingCPU (line3D.cc:925-950) + mutualOverlap (1086-1165): the four collinear points
// (projected src endpoints, tgt endpoints), score = |inner pair| / |outer pair| when the intervals touch at all.
// *valid = false when an intersection is degenerate (the reference skips the pair).
__device__ __forceinline__ float exact_overlap_f64(float4 qf, D3 e1, D3 e2, bool* valid)
{
    const D3 q1 = d3((double)qf.x, (double)qf.y, 1.0), q2 = d3((double)qf.z, (double)qf.w, 1.0);
    const D3 l2 = dcross(q1, q2);
    D3 a = dcross(l2, e1), b = dcross(l2, e2);
    *valid = fabs(a.z) > L3D_EPS_D && fabs(b.z) > L3D_EPS_D;
    if (!*valid) return 0.0f;
    a = d3(a.x / a.z, a.y / a.z, a.z / a.z);
    b = d3(b.x / b.z, b.y / b.z, b.z / b.z);
    const D3 cp[4] = {a, b, q1, q2};
    if (!(d_on_seg(cp[0], cp[2], cp[3]) || d_on_seg(cp[1], cp[2], cp[3]) || d_on_seg(cp[2], cp[0], cp[1]) || d_on_seg(cp[3], cp[0], cp[1])))
        return 0.0f;
    float max_dist = 0.0f; int o1 = 0, o2 = 3;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = i + 1; j < 4; ++j) {
            const float dist = (float)dnorm(dsub(cp[i], cp[j]));
            if (dist > max_dist) { max_dist = dist; o1 = i; o2 = j; }
        }
    if (max_dist < 1.0f) return 0.0f;
    int i1, i2;
    if (o1 == 0) { if (o2 == 1) { i1 = 2; i2 = 3; } else if (o2 == 2) { i1 = 1; i2 = 3; } else { i1 = 1; i2 = 2; } }
    else if (o1 == 1) { i1 = 0; i2 = o2 == 2 ? 3 : 2; }
    else { i1 = 0; i2 = 1; }
    D3 p = a, q = b;          // select without dynamically indexing cp[] (keeps it in registers)
    p = i1 == 0 ? a : (i1 == 1 ? b : q1);
    q = i2 == 1 ? b : (i2 == 2 ? q1 : q2);
    return (float)(dnorm(dsub(p, q)) / max_dist);
}

// the two triangulationDepths calls of matchingCPU (line3D.cc:953-964): d[0],d[1] src endpoints, d[2],d[3] tgt endpoints
__device__ __forceinline__ void exact_depths_f64(const SegRaysD& s, const SegRaysD& t, D3 Cs, D3 Ct, double* d)
{
    d[0] = d[1] = d[2] = d[3] = -1.0;
    if (!(fabs(ddot(s.r1, t.n)) < L3D_EPS_D || fabs(ddot(s.r2, t.n)) < L3D_EPS_D)) {
        d[0] = (ddot(Ct, t.n) - ddot(t.n, Cs)) / ddot(t.n, s.r1);
        d[1] = (ddot(Ct, t.n) - ddot(t.n, Cs)) / ddot(t.n, s.r2);
    }
    if (!(fabs(ddot(t.r1, s.n)) < L3D_EPS_D || fabs(ddot(t.r2, s.n)) < L3D_EPS_D)) {
        d[2] = (ddot(Cs, s.n) - ddot(s.n, Ct)) / ddot(s.n, t.r1);
        d[3] = (ddot(Cs, s.n) - ddot(s.n, Ct)) / ddot(s.n, t.r2);
    }
}
