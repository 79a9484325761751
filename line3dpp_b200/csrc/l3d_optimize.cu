// l3d_optimize.cu — bundling of the clustered 3D lines (SURVEY.md §8f-4): LineOptimizer::optimize (optimization.cc:8-303)
// with the cost functor LineReprojectionError (optimization.h:52-171).
//
// The reference builds a Ceres problem in which every camera and intrinsic block is constant (optimization.cc:178-188):
// only the four Cayley parameters (omega, s) of each line are free, the Jacobian is block diagonal and the SPARSE_SCHUR
// solve is one 4x4 system per line.  That is embarrassingly parallel, so the whole minimiser lives on the device:
//   k_opt_init       Pluecker -> Cayley per line (optimization.cc:34-91)
//   k_opt_linearize  per line: residuals with exact derivatives (forward-mode dual numbers, what AutoDiffCostFunction
//                    does), Huber loss through the Triggs corrector, cost, gradient J'r and J'J
//   k_opt_step       per line: Levenberg-Marquardt step on the Jacobi-scaled 4x4 system, model cost change, candidate
//                    point and its cost
//   k_opt_reduce     deterministic (fixed-order) sums of the per-line terms -> 8 doubles for the host
//   k_opt_finish     Cayley -> end points (optimization.cc:213-298)
// The host only plays Ceres' trust-region controller (ONE radius for the whole problem, accept / reject, tolerances) on
// those 8 numbers per iteration, so the iterates follow the reference solver's trajectory instead of a per-line variant:
// trust_region_minimizer.cc / levenberg_marquardt_strategy.cc defaults of ceres-solver 1.13-2.1 (radius 1e4, min relative
// decrease 1e-3, function / gradient / parameter tolerance 1e-6 / 1e-10 / 1e-8, Jacobi scaling fixed at iteration 0,
// diagonal clamped to [1e-6, 1e32]).  Ceres itself is a third-party dependency of the reference and is not part of its
// tree; parity is pinned on the reference's own before/after result fixtures (tests/golden/line3dpp_ref_opt_pairs_v1.npz).
// This file keeps nvcc's default FMA contraction off like the rest of the library (-fmad=false); nothing here is bit-pinned.
#include "l3d_ctx.cuh"
#include "l3d_device_f64.cuh"

#include <algorithm>
#include <cfloat>
#include <cmath>

namespace {

struct Jet4 { double a; double v[4]; };
__device__ __forceinline__ Jet4 J(double a) { Jet4 r; r.a = a; r.v[0] = r.v[1] = r.v[2] = r.v[3] = 0.0; return r; }
__device__ __forceinline__ Jet4 operator+(const Jet4& x, const Jet4& y) { Jet4 r; r.a = x.a + y.a; for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] + y.v[i]; return r; }
__device__ __forceinline__ Jet4 operator-(const Jet4& x, const Jet4& y) { Jet4 r; r.a = x.a - y.a; for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] - y.v[i]; return r; }
__device__ __forceinline__ Jet4 operator*(const Jet4& x, const Jet4& y) { Jet4 r; r.a = x.a * y.a; for (int i = 0; i < 4; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a; return r; }
__device__ __forceinline__ Jet4 operator*(double s, const Jet4& x) { Jet4 r; r.a = s * x.a; for (int i = 0; i < 4; ++i) r.v[i] = s * x.v[i]; return r; }
__device__ __forceinline__ Jet4 operator*(const Jet4& x, double s) { return s * x; }
__device__ __forceinline__ Jet4 operator/(const Jet4& x, const Jet4& y)
{ Jet4 r; const double inv = 1.0 / y.a, q = x.a * inv; r.a = q; for (int i = 0; i < 4; ++i) r.v[i] = (x.v[i] - q * y.v[i]) * inv; return r; }
__device__ __forceinline__ Jet4 jsqrt(const Jet4& x) { Jet4 r; r.a = sqrt(x.a); const double t = 1.0 / (2.0 * r.a); for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] * t; return r; }
__device__ __forceinline__ Jet4 jacos(const Jet4& x) { Jet4 r; r.a = acos(x.a); const double t = -1.0 / sqrt(1.0 - x.a * x.a); for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] * t; return r; }
__device__ __forceinline__ Jet4 jexp(const Jet4& x) { Jet4 r; r.a = exp(x.a); for (int i = 0; i < 4; ++i) r.v[i] = r.a * x.v[i]; return r; }
__device__ __forceinline__ bool jfinite(const Jet4& x) { bool f = isfinite(x.a); for (int i = 0; i < 4; ++i) f = f && isfinite(x.v[i]); return f; }

struct OptCam { double R[9], C[3], fx, fy, px, py; };          // 16 doubles, the layout of the `cams` argument
struct OptObs { double x1, y1, x2, y2, nx, ny; };              // end points + NORMAL of the observed 2D segment (optimization.cc:160-166)

#define OPT_PI 3.14159265358979323846
#define OPT_PI_2 1.57079632679489661923

// LineReprojectionError::operator() (optimization.h:66-162).  line = (omega, sx, sy, sz): Cayley parameters of the
// orthonormal Pluecker frame [Zhang & Koch 2014].  AngleAxisRotatePoint(angle-axis of R, m) == R m.
__device__ bool reprojection_error(const OptCam& cam, const OptObs& o, const Jet4 line[4], Jet4 res[2])
{
    const Jet4 omega = line[0], sx = line[1], sy = line[2], sz = line[3];
    const Jet4 nm = sx * sx + sy * sy + sz * sz;
    const Jet4 div = J(1.0) / (J(1.0) + nm);
    Jet4 l[3], m[3];
    l[0] = div * (J(1.0) - nm + 2.0 * sx * sx);
    l[1] = div * (2.0 * sz + 2.0 * sy * sx);
    l[2] = div * (-2.0 * sy + 2.0 * sz * sx);
    m[0] = omega * div * (-2.0 * sz + 2.0 * sx * sy);
    m[1] = omega * div * (J(1.0) - nm + 2.0 * sy * sy);
    m[2] = omega * div * (2.0 * sx + 2.0 * sz * sy);
    if (fabs(omega.a) < 1e-12) return false;
    m[0] = m[0] - (cam.C[1] * l[2] - cam.C[2] * l[1]);             // m - C x l: moment about the camera centre
    m[1] = m[1] + (cam.C[0] * l[2] - cam.C[2] * l[0]);
    m[2] = m[2] - (cam.C[0] * l[1] - cam.C[1] * l[0]);
    Jet4 q[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) q[i] = cam.R[3 * i] * m[0] + cam.R[3 * i + 1] * m[1] + cam.R[3 * i + 2] * m[2];
    Jet4 pl[3];                                                     // image line = cof(K) q
    pl[0] = cam.fy * q[0];
    pl[1] = cam.fx * q[1];
    pl[2] = (-cam.fy * cam.px) * q[0] - (cam.fx * cam.py) * q[1] + (cam.fx * cam.fy) * q[2];
    const Jet4 d = jsqrt(pl[0] * pl[0] + pl[1] * pl[1]);
    if (d.a < 1e-12) return false;
    Jet4 aw = J(1.0);                                               // angle weight exp(2 * angle to the observed direction)
    const Jet4 dx = pl[0] / d, dy = pl[1] / d;
    Jet4 angle = jacos(dx * o.nx + dy * o.ny);
    if (jfinite(angle)) {
        if (angle.a > OPT_PI_2) angle = J(OPT_PI) - angle;
        aw = jexp(2.0 * angle);
    }
    res[0] = (pl[0] * o.x1 + pl[1] * o.y1 + pl[2]) / d * aw;
    res[1] = (pl[0] * o.x2 + pl[1] * o.y2 + pl[2]) / d * aw;
    return true;
}

// cost 0.5 * sum rho(|r|^2), and (JAC) gradient J'r and J'J of the robustified blocks of one line.  HuberLoss(2)
// (LOSS_THRESHOLD, optimization.h:49): rho'' <= 0 everywhere, so Ceres' corrector scales residual and Jacobian by
// sqrt(rho') and nothing else.
template <bool JAC>
__device__ bool eval_line(const OptCam* __restrict__ cams, const int* __restrict__ res_cam, const OptObs* __restrict__ obs, long long r0, long long r1,
                          const double* x, double* cost, double* g, double* H)
{
    Jet4 line[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { line[k] = J(x[k]); line[k].v[k] = 1.0; }
    double c = 0.0;
    if (JAC) { for (int k = 0; k < 4; ++k) g[k] = 0.0; for (int k = 0; k < 10; ++k) H[k] = 0.0; }
    for (long long r = r0; r < r1; ++r) {
        Jet4 res[2];
        if (!reprojection_error(cams[res_cam[r]], obs[r], line, res)) return false;
        const double s = res[0].a * res[0].a + res[1].a * res[1].a;
        double rho = s, rho1 = 1.0;
        if (s > 4.0) { const double sr = sqrt(s); rho = 4.0 * sr - 4.0; rho1 = fmax(DBL_MIN, 2.0 / sr); }
        c += 0.5 * rho;
        if (JAC) {
            const double w = sqrt(rho1);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const double rr = w * res[e].a;
                double jr[4];
                for (int k = 0; k < 4; ++k) jr[k] = w * res[e].v[k];
                int idx = 0;
                for (int a = 0; a < 4; ++a) { g[a] += jr[a] * rr; for (int b = a; b < 4; ++b) H[idx++] += jr[a] * jr[b]; }
            }
        }
    }
    *cost = c;
    return true;
}

// (A + diag(D2)) y = b, A symmetric 4x4 as upper triangle (00 01 02 03 11 12 13 22 23 33); Cholesky
__device__ bool solve4(const double* A, const double* D2, const double* b, double* y)
{
    double M[4][4], Lc[4][4];
    int idx = 0;
    for (int a = 0; a < 4; ++a) for (int c = a; c < 4; ++c) { M[a][c] = M[c][a] = A[idx++]; }
    for (int a = 0; a < 4; ++a) M[a][a] += D2[a];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j <= i; ++j) {
            double s = M[i][j];
            for (int k = 0; k < j; ++k) s -= Lc[i][k] * Lc[j][k];
            if (i == j) { if (!(s > 0.0)) return false; Lc[i][i] = sqrt(s); } else Lc[i][j] = s / Lc[j][j];
        }
    double z[4];
    for (int i = 0; i < 4; ++i) { double s = b[i]; for (int k = 0; k < i; ++k) s -= Lc[i][k] * z[k]; z[i] = s / Lc[i][i]; }
    for (int i = 3; i >= 0; --i) { double s = z[i]; for (int k = i + 1; k < 4; ++k) s -= Lc[k][i] * y[k]; y[i] = s / Lc[i][i]; }
    return isfinite(y[0]) && isfinite(y[1]) && isfinite(y[2]) && isfinite(y[3]);
}

__global__ void __launch_bounds__(128)
k_opt_obs(long long nres, const double* __restrict__ res_xy, OptObs* __restrict__ obs)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nres) return;
    OptObs o;
    o.x1 = res_xy[4 * r]; o.y1 = res_xy[4 * r + 1]; o.x2 = res_xy[4 * r + 2]; o.y2 = res_xy[4 * r + 3];
    double dx = o.x2 - o.x1, dy = o.y2 - o.y1;
    const double n2 = dx * dx + dy * dy;
    if (n2 > 0) { const double n = sqrt(n2); dx /= n; dy /= n; }
    o.nx = -dy; o.ny = dx;                                           // direction as normal vector (optimization.cc:166)
    obs[r] = o;
}

// Pluecker -> Cayley (optimization.cc:34-91); isfree = 0: "symmetric line coords... do not bundle" or no residuals
__global__ void __launch_bounds__(128)
k_opt_init(int L, const double* __restrict__ p1p2, const long long* __restrict__ res_ptr, double* __restrict__ x, int* __restrict__ isfree)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    const double* p = p1p2 + 6 * i;
    const D3 P1 = d3(p[0], p[1], p[2]), P2 = d3(p[3], p[4], p[5]);
    const D3 l = dnormalized(d3(P2.x - P1.x, P2.y - P1.y, P2.z - P1.z));
    const D3 m = dcross(d3(0.5 * (P1.x + P2.x), 0.5 * (P1.y + P2.y), 0.5 * (P1.z + P2.z)), l);
    D3 e1, e2;
    if (dnorm(m) < 1e-12) {      // line through the origin of the working frame: any basis of the plane normal to l (the reference
        const D3 t = fabs(l.x) < 0.9 ? d3(1, 0, 0) : d3(0, 1, 0);   // takes Eigen's FullPivLU kernel; a set of measure zero)
        e1 = dnormalized(dcross(l, t)); e2 = dcross(l, e1);
    } else { e1 = dnormalized(m); e2 = dnormalized(dcross(l, m)); }
    // sx = (Q - I)(Q + I)^-1 with Q = [l e1 e2]
    const double Q[3][3] = {{l.x, e1.x, e2.x}, {l.y, e1.y, e2.y}, {l.z, e1.z, e2.z}};
    double A[3][3], B[3][3], Bi[3][3];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { A[r][c] = Q[r][c] - (r == c); B[r][c] = Q[r][c] + (r == c); }
    const double det = B[0][0] * (B[1][1] * B[2][2] - B[1][2] * B[2][1]) - B[0][1] * (B[1][0] * B[2][2] - B[1][2] * B[2][0]) +
                       B[0][2] * (B[1][0] * B[2][1] - B[1][1] * B[2][0]);
    const double id = 1.0 / det;
    Bi[0][0] = (B[1][1] * B[2][2] - B[1][2] * B[2][1]) * id; Bi[0][1] = (B[0][2] * B[2][1] - B[0][1] * B[2][2]) * id; Bi[0][2] = (B[0][1] * B[1][2] - B[0][2] * B[1][1]) * id;
    Bi[1][0] = (B[1][2] * B[2][0] - B[1][0] * B[2][2]) * id; Bi[1][1] = (B[0][0] * B[2][2] - B[0][2] * B[2][0]) * id; Bi[1][2] = (B[0][2] * B[1][0] - B[0][0] * B[1][2]) * id;
    Bi[2][0] = (B[1][0] * B[2][1] - B[1][1] * B[2][0]) * id; Bi[2][1] = (B[0][1] * B[2][0] - B[0][0] * B[2][1]) * id; Bi[2][2] = (B[0][0] * B[1][1] - B[0][1] * B[1][0]) * id;
    double S[3][3];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) S[r][c] = A[r][0] * Bi[0][c] + A[r][1] * Bi[1][c] + A[r][2] * Bi[2][c];
    double xi[4] = {dnorm(m), S[2][1], S[0][2], S[1][0]};
    const bool ok = !(isnan(xi[0]) || isnan(xi[1]) || isnan(xi[2]) || isnan(xi[3]));
    if (!ok) { xi[0] = -1.0; xi[1] = xi[2] = xi[3] = 0.0; }       // optimization.cc:72-84: kept constant, original end points survive
    for (int k = 0; k < 4; ++k) x[4 * i + k] = xi[k];
    isfree[i] = (ok && res_ptr[i + 1] > res_ptr[i]) ? 1 : 0;     // a block without residuals never enters the problem but is still written back
}

// per-line terms of one evaluation, reduced by k_opt_reduce:  part[0*L+i] cost  [1] |g|_inf  [2] failed
__global__ void __launch_bounds__(128)
k_opt_linearize(int L, const int* __restrict__ isfree, const OptCam* __restrict__ cams, const long long* __restrict__ res_ptr,
                const int* __restrict__ res_cam, const OptObs* __restrict__ obs, const double* __restrict__ x, double* __restrict__ g,
                double* __restrict__ H, double* __restrict__ part)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    double c = 0.0, gm = 0.0, fail = 0.0;
    if (isfree[i]) {
        double gi[4], Hi[10], xi[4] = {x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]};
        if (eval_line<true>(cams, res_cam, obs, res_ptr[i], res_ptr[i + 1], xi, &c, gi, Hi)) {
            for (int k = 0; k < 4; ++k) { g[4 * i + k] = gi[k]; gm = fmax(gm, fabs(gi[k])); }
            for (int k = 0; k < 10; ++k) H[10 * i + k] = Hi[k];
        } else { c = 0.0; fail = 1.0; }
    }
    part[i] = c; part[(size_t)L + i] = gm; part[2 * (size_t)L + i] = fail;
}

// Jacobi scaling, fixed at iteration zero: 1 / (1 + |column|)   (trust_region_minimizer.cc)
__global__ void __launch_bounds__(128) k_opt_scale(int L, const int* __restrict__ isfree, const double* __restrict__ H, double* __restrict__ S)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    const int DI[4] = {0, 4, 7, 9};
    for (int k = 0; k < 4; ++k) S[4 * i + k] = isfree[i] ? 1.0 / (1.0 + sqrt(H[10 * i + DI[k]])) : 1.0;
}

// LevenbergMarquardtStrategy::ComputeStep per 4x4 block + candidate point + candidate cost.
//   part[0] model cost change  [1] |step|^2  [2] |x|^2  [3] candidate cost  [4] solve failed  [5] candidate evaluation failed
__global__ void __launch_bounds__(128)
k_opt_step(int L, const int* __restrict__ isfree, const OptCam* __restrict__ cams, const long long* __restrict__ res_ptr, const int* __restrict__ res_cam,
           const OptObs* __restrict__ obs, const double* __restrict__ x, const double* __restrict__ g, const double* __restrict__ H,
           const double* __restrict__ S, double* __restrict__ diag, double radius, int reuse_diagonal, double* __restrict__ xc, double* __restrict__ part)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    double out[6] = {0, 0, 0, 0, 0, 0};
    if (isfree[i]) {
        const int DI[4] = {0, 4, 7, 9};
        double Hs[10], gs[4], D2[4], y[4], s[4], xi[4];
        for (int k = 0; k < 4; ++k) { s[k] = S[4 * i + k]; xi[k] = x[4 * i + k]; }
        int idx = 0;
        for (int a = 0; a < 4; ++a) { gs[a] = s[a] * g[4 * i + a]; for (int b = a; b < 4; ++b) { Hs[idx] = s[a] * s[b] * H[10 * i + idx]; ++idx; } }
        for (int k = 0; k < 4; ++k) {
            double dk = diag[4 * i + k];
            if (!reuse_diagonal) { dk = fmin(fmax(Hs[DI[k]], 1e-6), 1e32); diag[4 * i + k] = dk; }
            D2[k] = dk / radius;
        }
        if (solve4(Hs, D2, gs, y)) {
            double d[4], Hf[4][4];
            for (int k = 0; k < 4; ++k) d[k] = -y[k];
            idx = 0;
            for (int a = 0; a < 4; ++a) for (int b = a; b < 4; ++b) { Hf[a][b] = Hf[b][a] = Hs[idx++]; }
            double dg = 0.0, dHd = 0.0;
            for (int a = 0; a < 4; ++a) { double t = 0.0; for (int b = 0; b < 4; ++b) t += Hf[a][b] * d[b]; dHd += d[a] * t; dg += d[a] * gs[a]; }
            out[0] = -(dg + 0.5 * dHd);                             // -(J d)'(r + J d / 2)
            double cand[4];
            for (int k = 0; k < 4; ++k) { const double st = d[k] * s[k]; cand[k] = xi[k] + st; out[1] += st * st; out[2] += xi[k] * xi[k]; xc[4 * i + k] = cand[k]; }
            double cc;
            if (eval_line<false>(cams, res_cam, obs, res_ptr[i], res_ptr[i + 1], cand, &cc, nullptr, nullptr)) out[3] = cc; else out[5] = 1.0;
        } else out[4] = 1.0;
    }
    for (int k = 0; k < 6; ++k) part[(size_t)k * L + i] = out[k];
}

// totals[k] = sum (or max for MAXMASK bits) of part[k*L .. k*L+L) in a FIXED order: same bits on every run for a given L
__global__ void __launch_bounds__(1024) k_opt_reduce(int L, int nterms, unsigned int maxmask, const double* __restrict__ part, double* __restrict__ totals)
{
    __shared__ double sh[1024];
    for (int k = 0; k < nterms; ++k) {
        const bool mx = (maxmask >> k) & 1u;
        double acc = 0.0;
        for (int i = threadIdx.x; i < L; i += 1024) { const double v = part[(size_t)k * L + i]; acc = mx ? fmax(acc, v) : acc + v; }
        sh[threadIdx.x] = acc;
        __syncthreads();
        for (int o = 512; o > 0; o >>= 1) {
            if ((int)threadIdx.x < o) sh[threadIdx.x] = mx ? fmax(sh[threadIdx.x], sh[threadIdx.x + o]) : sh[threadIdx.x] + sh[threadIdx.x + o];
            __syncthreads();
        }
        if (threadIdx.x == 0) totals[k] = sh[0];
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_opt_accept(long long n, const int* __restrict__ isfree, const double* __restrict__ xc, double* __restrict__ x)
{
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n && isfree[j >> 2]) x[j] = xc[j];
}

// Cayley -> end points around the old mid point (optimization.cc:213-291); valid = 0 if the segment has no length (293-298)
__global__ void __launch_bounds__(128)
k_opt_finish(int L, const double* __restrict__ x, const double* __restrict__ p_old, double* __restrict__ p_out, int* __restrict__ valid)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    const double* o = p_old + 6 * i;
    D3 P1 = d3(o[0], o[1], o[2]), P2 = d3(o[3], o[4], o[5]);
    const double omega = x[4 * i];
    if (!(omega < 0.0 || fabs(omega) < 1e-12)) {
        const double s0 = x[4 * i + 1], s1 = x[4 * i + 2], s2 = x[4 * i + 3], nm = s0 * s0 + s1 * s1 + s2 * s2, f = 1.0 / (1.0 + nm);
        // columns 0 and 1 of Q = f ((1 - nm) I + 2 [s]x + 2 s s')
        const D3 l = d3(f * ((1.0 - nm) + 2.0 * s0 * s0), f * (2.0 * s2 + 2.0 * s1 * s0), f * (-2.0 * s1 + 2.0 * s2 * s0));
        const D3 m = d3(omega * f * (-2.0 * s2 + 2.0 * s0 * s1), omega * f * ((1.0 - nm) + 2.0 * s1 * s1), omega * f * (2.0 * s0 + 2.0 * s2 * s1));
        if (fabs(l.x) > 1e-12 || fabs(l.y) > 1e-12 || fabs(l.z) > 1e-12) {
            const D3 Pm = d3(0.5 * (P1.x + P2.x), 0.5 * (P1.y + P2.y), 0.5 * (P1.z + P2.z));
            double x1, x2, x3;
            if (fabs(l.x) > fabs(l.y) && fabs(l.x) > fabs(l.z)) { x1 = Pm.x; x3 = (-m.y - x1 * l.z) / -l.x; x2 = (m.z - x1 * l.y) / -l.x; }
            else if (fabs(l.y) > fabs(l.x) && fabs(l.y) > fabs(l.z)) { x2 = Pm.y; x3 = (m.x - x2 * l.z) / -l.y; x1 = (m.z + x2 * l.x) / l.y; }
            else { x3 = Pm.z; x2 = (m.x + x3 * l.y) / l.z; x1 = (-m.y + x3 * l.x) / l.z; }
            P1 = d3(x1 + l.x, x2 + l.y, x3 + l.z); P2 = d3(x1 - l.x, x2 - l.y, x3 - l.z);
        }
    }
    double* q = p_out + 6 * i;
    q[0] = P1.x; q[1] = P1.y; q[2] = P1.z; q[3] = P2.x; q[4] = P2.y; q[5] = P2.z;
    valid[i] = dnorm(d3(P1.x - P2.x, P1.y - P2.y, P1.z - P2.z)) > 1e-12 ? 1 : 0;
}

}  // namespace

extern "C" {

// LineOptimizer::optimize for `num_lines` clustered 3D lines.  p1p2: 6 doubles per line (cluster segment, working frame);
// res_ptr[num_lines + 1] / res_cam / res_xy: the 2D residuals of every line (camera index into `cams`, float segment
// coordinates x1 y1 x2 y2 as doubles); cams: 16 doubles per camera (R row-major, C, fx, fy, px, py), all constant.
// p1p2_out (may alias p1p2) and valid_out per line (0 = the reference drops the cluster).  summary (optional, 8 doubles):
// iterations, initial cost, final cost, termination (0 convergence, 1 max_iter, 2 failure), successful steps, free lines,
// final trust-region radius, kernels launched.
int l3d_optimize_lines(l3d_ctx* c, int num_lines, const double* p1p2, const long long* res_ptr, const int32_t* res_cam, const double* res_xy,
                       int num_cams, const double* cams, int max_iter, double* p1p2_out, int32_t* valid_out, double* summary)
{
    if (!c || num_lines < 0 || num_cams < 0 || (num_lines && (!p1p2 || !res_ptr || !p1p2_out || !valid_out))) return l3d_fail(c, L3D_ERR_INVALID, "l3d_optimize_lines: bad arguments");
    if (summary) for (int k = 0; k < 8; ++k) summary[k] = 0.0;
    if (num_lines == 0) return L3D_OK;
    const int L = num_lines;
    if (res_ptr[0] != 0) return l3d_fail(c, L3D_ERR_INVALID, "l3d_optimize_lines: res_ptr[0] must be 0");
    for (int i = 0; i < L; ++i)
        if (res_ptr[i + 1] < res_ptr[i]) return l3d_fail(c, L3D_ERR_INVALID, "l3d_optimize_lines: res_ptr must not decrease");
    const long long NR = res_ptr[L];
    if (NR && (!res_cam || !res_xy || !cams || num_cams == 0)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_optimize_lines: bad residual arrays");
    for (long long r = 0; r < NR; ++r) if (res_cam[r] < 0 || res_cam[r] >= num_cams) return l3d_fail(c, L3D_ERR_INVALID, "l3d_optimize_lines: camera index out of range");
    cudaSetDevice(c->device);
    OptState& O = c->opt;
    int rc;
    L3D_RESERVE(O.d_obs, (long long)sizeof(OptObs) * NR, "opt observations");
    L3D_RESERVE(O.d_x, 32ll * L, "opt x"); L3D_RESERVE(O.d_xc, 32ll * L, "opt x candidate"); L3D_RESERVE(O.d_g, 32ll * L, "opt gradient");
    L3D_RESERVE(O.d_H, 80ll * L, "opt JtJ"); L3D_RESERVE(O.d_S, 32ll * L, "opt scaling"); L3D_RESERVE(O.d_diag, 32ll * L, "opt diagonal"); L3D_RESERVE(O.d_free, 4ll * L, "opt free flags");
    L3D_RESERVE(O.d_part, 48ll * L, "opt partial sums"); L3D_RESERVE(O.d_tot, 64, "opt totals");
    // without residuals, res_cam, res_xy and cams may be null: their blocks are empty and not uploaded
    HostBlock in[5] = {host_array(p1p2, 48ull * L), host_array(res_ptr, 8ull * (L + 1)), host_array(res_cam, 4ull * NR), host_array(res_xy, 32ull * NR),
                       host_array(cams, NR ? 128ull * num_cams : 0)};
    HostBlock out[2] = {host_array(p1p2_out, 48ull * L), host_array(valid_out, 4ull * L)};
    if ((rc = l3d_stage_host(c, in, 5, out, 2))) return rc;
    cudaStream_t st = c->stream;
    const unsigned int nbl = (unsigned int)((L + 127) / 128);
    long long launches = 0;
    if (NR) { k_opt_obs<<<(unsigned int)((NR + 127) / 128), 128, 0, st>>>(NR, (const double*)in[3].dev, (OptObs*)O.d_obs.p); ++launches; }
    k_opt_init<<<nbl, 128, 0, st>>>(L, (const double*)in[0].dev, (const long long*)in[1].dev, (double*)O.d_x.p, (int*)O.d_free.p); ++launches;
    const int* isfree = (const int*)O.d_free.p;
    const OptCam* dcams = (const OptCam*)in[4].dev; const OptObs* dobs = (const OptObs*)O.d_obs.p;
    const long long* dptr = (const long long*)in[1].dev; const int* dcam = (const int*)in[2].dev;
    double* x = (double*)O.d_x.p; double* xc = (double*)O.d_xc.p; double* part = (double*)O.d_part.p; double* tot = (double*)O.d_tot.p;
    double h[8];
    auto totals = [&](int nterms, unsigned int maxmask) -> int {
        k_opt_reduce<<<1, 1024, 0, st>>>(L, nterms, maxmask, part, tot); ++launches;
        L3D_CUDA(c, cudaMemcpyAsync(h, tot, 8 * (size_t)nterms, cudaMemcpyDeviceToHost, st), "opt totals");
        L3D_CUDA(c, cudaStreamSynchronize(st), "opt iteration");
        return L3D_OK;
    };
    auto linearize = [&]() -> int {
        k_opt_linearize<<<nbl, 128, 0, st>>>(L, isfree, dcams, dptr, dcam, dobs, x, (double*)O.d_g.p, (double*)O.d_H.p, part); ++launches;
        return totals(3, 0x2u);                                      // cost (sum), |g|_inf (max), failures (sum)
    };
    // free lines
    {
        std::vector<int> fr((size_t)L);
        L3D_CUDA(c, cudaMemcpyAsync(fr.data(), O.d_free.p, 4ull * L, cudaMemcpyDeviceToHost, st), "opt free flags");
        L3D_CUDA(c, cudaStreamSynchronize(st), "opt init");
        long long nfree = 0; for (int v : fr) nfree += v;
        if (summary) summary[5] = (double)nfree;
        if (nfree == 0) max_iter = -1;
    }
    int term = 0, it = 0, nsucc = 0;
    double cost = 0.0, cost0 = 0.0, radius = 1e4;
    if (max_iter >= 0) {
        if ((rc = linearize())) return rc;
        if (h[2] > 0.0) term = 2;                                    // initial evaluation failed: nothing is changed, no cost reported
        else {
            cost = cost0 = h[0];
            k_opt_scale<<<nbl, 128, 0, st>>>(L, isfree, (const double*)O.d_H.p, (double*)O.d_S.p); ++launches;
            double decrease_factor = 2.0; bool reuse_diagonal = false; int invalid = 0;
            bool done = h[1] <= 1e-10;                               // gradient tolerance at iteration zero
            while (!done) {
                if (it >= max_iter) { term = 1; break; }
                if (radius <= 1e-32) break;                          // minimum trust-region radius: convergence
                ++it;
                k_opt_step<<<nbl, 128, 0, st>>>(L, isfree, dcams, dptr, dcam, dobs, x, (const double*)O.d_g.p, (const double*)O.d_H.p, (const double*)O.d_S.p,
                                                (double*)O.d_diag.p, radius, reuse_diagonal ? 1 : 0, xc, part); ++launches;
                if ((rc = totals(6, 0u))) return rc;
                reuse_diagonal = true;
                const double model_change = h[0], step_sq = h[1], x_sq = h[2];
                if (h[4] > 0.0 || !(model_change > 0.0)) {           // HandleInvalidStep
                    if (++invalid >= 5) { term = 2; break; }
                    radius *= 0.5; reuse_diagonal = false;
                    continue;
                }
                invalid = 0;
                const double cand = h[5] > 0.0 ? DBL_MAX : h[3];
                if (std::sqrt(step_sq) <= 1e-8 * (std::sqrt(x_sq) + 1e-8)) break;              // parameter tolerance
                if (std::fabs(cost - cand) <= 1e-6 * cost) break;                               // function tolerance (candidate not applied)
                const double quality = (cost - cand) / model_change;
                if (quality > 1e-3) {                                // HandleSuccessfulStep
                    k_opt_accept<<<(unsigned int)((4ll * L + 255) / 256), 256, 0, st>>>(4ll * L, isfree, xc, x); ++launches;
                    ++nsucc;
                    if ((rc = linearize())) return rc;
                    if (h[2] > 0.0) { term = 2; break; }
                    cost = h[0];
                    radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * quality - 1.0, 3)));
                    decrease_factor = 2.0; reuse_diagonal = false;
                    if (h[1] <= 1e-10) break;                        // gradient tolerance
                } else {                                             // HandleUnsuccessfulStep
                    radius /= decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true;
                }
            }
        }
    }
    k_opt_finish<<<nbl, 128, 0, st>>>(L, x, (const double*)in[0].dev, (double*)out[0].dev, (int*)out[1].dev); ++launches;
    L3D_CUDA(c, cudaGetLastError(), "opt kernels");
    if ((rc = l3d_unstage_host(c, out, 2, "opt"))) return rc;
    c->launches += launches;
    if (summary) { summary[0] = it; summary[1] = cost0; summary[2] = cost; summary[3] = term; summary[4] = nsucc; summary[6] = radius; summary[7] = (double)launches; }
    return L3D_OK;
}

}  // extern "C"
