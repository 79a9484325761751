// l3d_undistort.cu — lens undistortion of 8-bit images: what Line3D::undistortImage computes with OpenCV (line3D.cc:83-109,
// initUndistortRectifyMap with fixed-point CV_16SC2 + CV_16UC1 maps, then remap INTER_LINEAR / BORDER_CONSTANT 0), the undistortion of
// points as cv::undistortPoints / cv::fisheye::undistortPoints compute it, and the four C-ABI entry points declared in include/l3d_capi.h.  Two lens models: OpenCV's standard one with up to 8 coefficients (radtan) and
// cv::fisheye's.  The output may have its own camera matrix and size (OpenCV's newCameraMatrix / newImageSize).  The arithmetic contract is DESIGN.md §4a; tests/undistort_model.py and tests/lens_model.py restate it.
//
// None of these calls belongs to the pipeline: they never drop a stage and touch only the buffers of UndistortState and, in host
// mode, the context's staging pair.
#include "l3d_ctx.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#define UD_TW 128       // columns per tile of k_undistort_u8 (one per thread)
#define UD_TH 16        // rows per tile

// the kernels' lens kinds (L3DUndistImage::kind): radtan without and with the rational denominator, fisheye.  Each has its own
// instance of k_undistort_u8, so the pinhole kernel keeps its 48 registers (a double division or atan in the same kernel costs 16 / 24).
enum { UD_RADTAN = 0, UD_RATIONAL = 1, UD_FISHEYE = 2, UD_KINDS = 3 };

// cvRound(t * 32) as OpenCV's x86 build does it: round half to even; a value that is not finite or does not fit int32 gives INT_MIN
__device__ __forceinline__ int ud_fix(double t)
{
    const double r = rint(t * 32.0);
    return (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;
}

// Fixed-point source position (u*32, v*32) of the output pixel whose normalised coordinates are x = ir2 + j*ir0, y = i*ir4 + ir5
// (ir: the inverse of the new camera matrix; its zero entries only add signed zeros), projected with the camera's fx, fy, cx, cy.  x2 = x*x and y2 = y*y come from the caller so that a tile computes them once
// per column / row.  Terms whose coefficients are zero are skipped: that changes at most the sign of a zero, which the rounding
// erases.  Plain IEEE double operations in the reference's order (the library is compiled with -fmad=false).
template <bool RATIONAL>
__device__ __forceinline__ void ud_map_point(const L3DUndistImage& d, double x, double x2, double y, double y2, int& iu, int& iv)
{
    const double r2 = x2 + y2;
    double kr = 1.0 + (d.full_radial ? ((d.k3 * r2 + d.k2) * r2 + d.k1) : d.k1) * r2;
    if (RATIONAL) kr = kr / (1.0 + ((d.k6 * r2 + d.k5) * r2 + d.k4) * r2);
    double xd = x * kr, yd = y * kr;
    if (d.tangential) {
        const double _2xy = 2.0 * x * y;
        xd = xd + d.p1 * _2xy + d.p2 * (r2 + 2.0 * x2);
        yd = yd + d.p1 * (r2 + 2.0 * y2) + d.p2 * _2xy;
    }
    iu = ud_fix(d.fx * xd + d.cx);
    iv = ud_fix(d.fy * yd + d.cy);
}

// The same for cv::fisheye::initUndistortRectifyMap with R = I, P = newK: x comes from the column table (OpenCV's loop accumulates it),
// r = |(x, y)|, theta = atan(r), theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8), u = fx x (theta_d / r) + cx.
// Everything but atan is IEEE; atan may differ from the host's in the last ulp (the fisheye contract is one step, DESIGN.md §4a).
__device__ __forceinline__ void ud_fisheye_point(const L3DUndistImage& d, double x, double x2, double y, double y2, int& iu, int& iv)
{
    const double r = sqrt(x2 + y2);
    const double th = atan(r);
    const double t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
    const double thd = th * (1.0 + d.k1 * t2 + d.k2 * t4 + d.k3 * t6 + d.k4 * t8);
    const double scale = r == 0.0 ? 1.0 : thd / r;
    iu = ud_fix(d.fx * x * scale + d.cx);
    iv = ud_fix(d.fy * y * scale + d.cy);
}

__device__ __forceinline__ short ud_sat16(int v) { return (short)max(-32768, min(32767, v)); }

// OpenCV's map entry: integer pixel and the 1/32-px fractions packed as ty*32 + tx.  The pixel is saturated to int16 by
// initUndistortRectifyMap and truncated (wraps) by the fisheye loop's (short) cast.
template <int KIND>
__device__ __forceinline__ void ud_entry(int iu, int iv, short2& xy, unsigned short& frac)
{
    if (KIND == UD_FISHEYE) xy = make_short2((short)(iu >> 5), (short)(iv >> 5));
    else xy = make_short2(ud_sat16(iu >> 5), ud_sat16(iv >> 5));
    frac = (unsigned short)(((iv & 31) << 5) + (iu & 31));
}

// source position and map entry of one destination pixel under the image's model
template <int KIND>
__device__ __forceinline__ void ud_map_entry(const L3DUndistImage& d, double x, double x2, double y, double y2, short2& xy, unsigned short& frac)
{
    int iu, iv;
    if (KIND == UD_FISHEYE) ud_fisheye_point(d, x, x2, y, y2, iu, iv);
    else ud_map_point<KIND == UD_RATIONAL>(d, x, x2, y, y2, iu, iv);
    ud_entry<KIND>(iu, iv, xy, frac);
}

// x of column j: j*ir0 + ir2 (radtan) or the fisheye column table
template <int KIND>
__device__ __forceinline__ double ud_column_x(const L3DUndistImage& d, int j)
{
    return KIND == UD_FISHEYE ? d.xcol[j] : (double)j * d.ir0 + d.ir2;
}

// remap's bilinear tap sum for one destination pixel: weights (32-tx|tx)*(32-ty|ty)*32 sum to 32768; a tap outside the image
// reads the border value 0; result (sum + 16384) >> 15 clamped to 8 bits
template <int C>
__device__ __forceinline__ void ud_tap_sum(const unsigned char* __restrict__ src, long long pitch, int W, int H, short2 xy, unsigned short frac,
                                           unsigned char* __restrict__ out)
{
    const int tx = frac & 31, ty = frac >> 5;
    const int w[4] = {(32 - tx) * (32 - ty) * 32, tx * (32 - ty) * 32, (32 - tx) * ty * 32, tx * ty * 32};
    int acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int X = xy.x + (t & 1), Y = xy.y + (t >> 1);
        if ((unsigned)X < (unsigned)W && (unsigned)Y < (unsigned)H) {
            const unsigned char* p = src + (long long)Y * pitch + (long long)X * C;
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] += w[t] * (int)__ldg(p + c);
        }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) out[c] = (unsigned char)max(0, min(255, (acc[c] + 16384) >> 15));
}

// the maps of one image, OpenCV's layout: map_xy short2[oH*oW], map_frac ushort[oH*oW] over the output grid, rows packed
template <int KIND>
__global__ void __launch_bounds__(UD_TW) k_undistort_map(L3DUndistImage d, short2* __restrict__ map_xy, unsigned short* __restrict__ map_frac)
{
    const int j = blockIdx.x * UD_TW + threadIdx.x, i = blockIdx.y;
    if (j >= d.out_width) return;
    const double y = (double)i * d.ir4 + d.ir5;
    const long long o = (long long)i * d.out_width + j;
    const double x = ud_column_x<KIND>(d, j);
    ud_map_entry<KIND>(d, x, x * x, y, y * y, map_xy[o], map_frac[o]);
}

// remap of one image with caller-given maps (same layout, output grid); the taps are bounded by the source size
template <int C>
__global__ void __launch_bounds__(UD_TW) k_remap_u8(L3DUndistImage d, const short2* __restrict__ map_xy, const unsigned short* __restrict__ map_frac)
{
    const int j = blockIdx.x * UD_TW + threadIdx.x, i = blockIdx.y;
    if (j >= d.out_width) return;
    const long long o = (long long)i * d.out_width + j;
    ud_tap_sum<C>(d.src, d.src_pitch, d.width, d.height, map_xy[o], map_frac[o], d.dst + (long long)i * d.dst_pitch + (long long)j * C);
}

template <int KIND, int C>
__device__ __forceinline__ void ud_tile_rows(const L3DUndistImage& d, int j, int i0, int rows, const double2* s_y)
{
    const double x = ud_column_x<KIND>(d, j), x2 = x * x;
    unsigned char* out = d.dst + (long long)i0 * d.dst_pitch + (long long)j * C;
    for (int r = 0; r < rows; ++r, out += d.dst_pitch) {
        short2 xy; unsigned short frac;
        ud_map_entry<KIND>(d, x, x2, s_y[r].x, s_y[r].y, xy, frac);
        ud_tap_sum<C>(d.src, d.src_pitch, d.width, d.height, xy, frac, out);
    }
}

// One CTA's work of k_undistort_u8: UD_TW output columns x UD_TH output rows of the image d (the taps are bounded by its source size)
template <int KIND>
__device__ __forceinline__ void ud_tile(const L3DUndistImage& d, double2* s_y)
{
    const long long t = (long long)blockIdx.x - d.tile0;
    const int i0 = (int)(t / d.tiles_x) * UD_TH, j = (int)(t % d.tiles_x) * UD_TW + threadIdx.x;
    if (threadIdx.x < UD_TH) {
        const double y = (double)(i0 + threadIdx.x) * d.ir4 + d.ir5;
        s_y[threadIdx.x] = make_double2(y, y * y);
    }
    __syncthreads();
    if (j >= d.out_width) return;
    const int rows = min(UD_TH, d.out_height - i0);
    if (d.channels == 3) ud_tile_rows<KIND, 3>(d, j, i0, rows, s_y);
    else ud_tile_rows<KIND, 1>(d, j, i0, rows, s_y);
}

// The fused hot path over a batch: map entries in registers, never stored.  One CTA = UD_TW columns x UD_TH rows of one image's
// output grid; the tiles of all images of one model form one grid (image found by binary search over tile0), grey and RGB images
// alike.  One instance per lens kind (UD_RADTAN ..), each over its own images.  The pinhole and fisheye instances hold the descriptor
// in registers (48 and 55).  The rational one would need 72 that way; it reads the descriptor from a shared-memory copy instead, which
// the compiler reloads where it is used (the output may alias it as far as the compiler knows), and stays below 64.
template <int KIND>
__global__ void __launch_bounds__(UD_TW) k_undistort_u8(const L3DUndistImage* __restrict__ imgs, int n)
{
    __shared__ double2 s_y[UD_TH];          // (y, y*y) of the tile's rows
    const L3DUndistImage* g = imgs + last_le(n, (long long)blockIdx.x, [&](int i) { return imgs[i].tile0; });
    if (KIND == UD_RATIONAL) {
        __shared__ L3DUndistImage s_d;
        static_assert(sizeof(L3DUndistImage) % 8 == 0 && sizeof(L3DUndistImage) / 8 <= UD_TW, "descriptor staging");
        if (threadIdx.x < sizeof(L3DUndistImage) / 8) ((long long*)&s_d)[threadIdx.x] = __ldg((const long long*)g + threadIdx.x);
        __syncthreads();
        ud_tile<KIND>(s_d, s_y);
    } else {
        const L3DUndistImage d = *g;
        ud_tile<KIND>(d, s_y);
    }
}

// ------------------------------------------------------------------------------------------------ points
// cv::undistortPoints(src, dst, K, D, noArray(), P) of one point: cvUndistortPointsInternal with TermCriteria(COUNT, 5, 0.01), so five
// fixed-point steps and no reprojection error.  The identity tilt (invMatTilt) and rectification (RR = P * I) products are spelled
// out as cv::Matx and cvMatMul sum them: they add only signed zeros to finite values, but make an infinite coordinate NaN.
__device__ __forceinline__ void up_radtan(const L3DPointSet& s, double u, double v, double& X, double& Y)
{
    const double* k = s.k;
    double x = (u - s.cx) * s.ifx, y = (v - s.cy) * s.ify;
    const double tx = ((0.0 + 1.0 * x) + 0.0 * y) + 0.0 * 1.0, ty = ((0.0 + 0.0 * x) + 1.0 * y) + 0.0 * 1.0;
    const double tz = ((0.0 + 0.0 * x) + 0.0 * y) + 1.0 * 1.0, inv = tz != 0.0 ? 1.0 / tz : 1.0;
    const double x0 = inv * tx, y0 = inv * ty;
    x = x0; y = y0;
    for (int j = 0; j < 5; ++j) {
        const double r2 = x * x + y * y;
        const double icdist = (1.0 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1.0 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
        if (icdist < 0.0) {                 // OpenCV's regression_14583 fallback: the point as if there were no distortion
            x = (u - s.cx) * s.ifx;
            y = (v - s.cy) * s.ify;
            break;
        }
        // k[8..11] (thin prism) are zero; their products stay, for the NaN an infinite r2 gives
        const double dx = (((2.0 * k[2]) * x) * y + k[3] * (r2 + (2.0 * x) * x) + 0.0 * r2) + (0.0 * r2) * r2;
        const double dy = ((k[2] * (r2 + (2.0 * y) * y) + ((2.0 * k[3]) * x) * y) + 0.0 * r2) + (0.0 * r2) * r2;
        x = (x0 - dx) * icdist;
        y = (y0 - dy) * icdist;
    }
    const double xx = (s.nfx * x + 0.0 * y) + s.ncx, yy = (0.0 * x + s.nfy * y) + s.ncy;
    const double ww = 1.0 / ((0.0 * x + 0.0 * y) + 1.0);
    X = xx * ww; Y = yy * ww;
}

// cv::fisheye::undistortPoints(src, dst, K, D, I, P) of one point with its default TermCriteria(MAX_ITER + EPS, 10, 1e-8).  tan is the
// device's (within an ulp or two of glibc's); the rest is IEEE double in OpenCV's order.
__device__ __forceinline__ void up_fisheye(const L3DPointSet& s, double u, double v, double& X, double& Y)
{
    const double* k = s.k;
    const double pwx = (u - s.cx) / s.fx, pwy = (v - s.cy) / s.fy;
    const double hp = 3.14159265358979323846 / 2.0;
    double td = sqrt(pwx * pwx + pwy * pwy);
    td = -hp < td ? td : -hp;               // std::max(-pi/2, td): NaN becomes -pi/2
    td = hp < td ? hp : td;                 // std::min(td, pi/2)
    double theta = td, scale = 0.0;
    bool converged = true;
    if (fabs(td) > 1e-8) {
        converged = false;
        for (int j = 0; j < 10; ++j) {
            const double t2 = theta * theta, t4 = t2 * t2, t6 = t4 * t2, t8 = t6 * t2;
            const double a = k[0] * t2, b = k[1] * t4, c = k[2] * t6, d = k[3] * t8;
            const double fix = (theta * (1.0 + a + b + c + d) - td) / (1.0 + 3.0 * a + 5.0 * b + 7.0 * c + 9.0 * d);
            theta = theta - fix;
            if (fabs(fix) < 1e-8) { converged = true; break; }
        }
        scale = tan(theta) / td;
    }
    const bool flipped = (td < 0.0 && theta > 0.0) || (td > 0.0 && theta < 0.0);
    if (!converged || flipped) { X = -1000000.0; Y = -1000000.0; return; }
    const double px = pwx * scale, py = pwy * scale;
    const double rx = ((0.0 + s.nfx * px) + 0.0 * py) + s.ncx * 1.0, ry = ((0.0 + 0.0 * px) + s.nfy * py) + s.ncy * 1.0;
    const double rz = ((0.0 + 0.0 * px) + 0.0 * py) + 1.0 * 1.0;
    X = rx / rz; Y = ry / rz;
}

// one thread per point of all sets; a set is found by binary search over p0.  src and dst may be the same array (each thread reads
// its point before it writes it).
#define UP_THREADS 256
__global__ void __launch_bounds__(UP_THREADS) k_undistort_points(const L3DPointSet* __restrict__ sets, int n, long long total)
{
    const long long i = (long long)blockIdx.x * UP_THREADS + threadIdx.x;
    if (i >= total) return;
    const L3DPointSet& s = sets[last_le(n, i, [&](int j) { return sets[j].p0; })];
    const long long q = 2 * (i - s.p0);
    const double u = s.src[q], v = s.src[q + 1];
    double X, Y;
    if (s.fisheye) up_fisheye(s, u, v, X, Y);
    else up_radtan(s, u, v, X, Y);
    s.dst[q] = (float)X;
    s.dst[q + 1] = (float)Y;
}

// ------------------------------------------------------------------------------------------------ host side
// the camera, lens and new-K checks of one descriptor
static int ud_check_camera(l3d_ctx* c, const l3d_undistort_desc& u, const char* what)
{
    char buf[160];
    auto bad = [&](const char* why) { snprintf(buf, sizeof(buf), "%s: %s", what, why); return l3d_fail(c, L3D_ERR_INVALID, buf); };
    if (!std::isfinite(u.fx) || !std::isfinite(u.fy) || u.fx == 0.0 || u.fy == 0.0) return bad("fx and fy must be finite and non-zero");
    bool finite = std::isfinite(u.cx) && std::isfinite(u.cy), zero = true;
    for (int k = 0; k < 3; ++k) { finite = finite && std::isfinite(u.radial[k]) && std::isfinite(u.rational[k]); zero = zero && u.radial[k] == 0.0 && u.rational[k] == 0.0; }
    for (int k = 0; k < 2; ++k) { finite = finite && std::isfinite(u.tangential[k]); zero = zero && u.tangential[k] == 0.0; }
    for (int k = 0; k < 4; ++k) finite = finite && std::isfinite(u.fisheye[k]);
    if (!finite) return bad("principal point and coefficients must be finite");
    if (u.model != L3D_LENS_RADTAN && u.model != L3D_LENS_FISHEYE) return bad("unknown lens model");
    if (u.model == L3D_LENS_FISHEYE && !zero) return bad("a fisheye lens takes no radial, tangential or rational coefficients");
    const bool new_k = u.new_fx != 0.0 || u.new_fy != 0.0 || u.new_cx != 0.0 || u.new_cy != 0.0;
    if (new_k && (!std::isfinite(u.new_fx) || !std::isfinite(u.new_fy) || u.new_fx == 0.0 || u.new_fy == 0.0))
        return bad("new_fx and new_fy must be finite and non-zero");
    if (new_k && (!std::isfinite(u.new_cx) || !std::isfinite(u.new_cy))) return bad("new_cx and new_cy must be finite");
    return L3D_OK;
}

// checks one descriptor; `image`: the pixel pointers and pitches are used, `camera`: the intrinsics and coefficients are used
static int ud_check(l3d_ctx* c, const l3d_undistort_desc& u, bool image, bool camera, const char* what)
{
    char buf[160];
    auto bad = [&](const char* why) { snprintf(buf, sizeof(buf), "%s: %s", what, why); return l3d_fail(c, L3D_ERR_INVALID, buf); };
    if (u.width < 1 || u.width > 32767 || u.height < 1 || u.height > 32767) return bad("width and height must lie in [1, 32767]");
    if (u.channels != 1 && u.channels != 3) return bad("channels must be 1 or 3");
    if ((u.out_width != 0 || u.out_height != 0) && (u.out_width < 1 || u.out_width > 32767 || u.out_height < 1 || u.out_height > 32767))
        return bad("out_width and out_height must both be 0 or lie in [1, 32767]");
    if (image) {
        if (u.src_pitch < (long long)u.width * u.channels) return bad("row pitch below width * channels");
        if (u.dst_pitch < (long long)(u.out_width ? u.out_width : u.width) * u.channels) return bad("dst row pitch below out_width * channels");
        if (!u.src || !u.dst) return bad("null image pointer");
        if (u.src == u.dst) return bad("src == dst (no in-place undistortion)");
    }
    return camera ? ud_check_camera(c, u, what) : L3D_OK;
}

// kernel parameters of one point set (the new K: the camera's own when new_fx .. new_cy are all zero)
static L3DPointSet up_set(const l3d_undistort_desc& u, const float* src, float* dst, long long p0)
{
    L3DPointSet s;
    memset(&s, 0, sizeof(s));
    s.src = src; s.dst = dst; s.p0 = p0;
    s.fx = u.fx; s.fy = u.fy; s.cx = u.cx; s.cy = u.cy; s.ifx = 1.0 / u.fx; s.ify = 1.0 / u.fy;
    const bool new_k = u.new_fx != 0.0 || u.new_fy != 0.0 || u.new_cx != 0.0 || u.new_cy != 0.0;
    s.nfx = new_k ? u.new_fx : u.fx; s.nfy = new_k ? u.new_fy : u.fy; s.ncx = new_k ? u.new_cx : u.cx; s.ncy = new_k ? u.new_cy : u.cy;
    s.fisheye = u.model == L3D_LENS_FISHEYE;
    if (s.fisheye) {
        for (int i = 0; i < 4; ++i) s.k[i] = u.fisheye[i];
    } else {
        const double k[8] = {u.radial[0], u.radial[1], u.tangential[0], u.tangential[1], u.radial[2], u.rational[0], u.rational[1], u.rational[2]};
        memcpy(s.k, k, sizeof(k));
    }
    return s;
}

static int ud_out_width(const l3d_undistort_desc& u) { return u.out_width ? u.out_width : u.width; }
static int ud_out_height(const l3d_undistort_desc& u) { return u.out_height ? u.out_height : u.height; }

// kernel parameters of one image; the inverse of the new camera matrix (the camera's own K when new_fx .. new_cy are all zero) is
// formed like OpenCV's 3x3 inversion (cofactors / determinant).  cv::fisheye inverts by SVD instead, which can differ in the last
// bits; DESIGN.md §4a counts what that costs.
static L3DUndistImage ud_image(const l3d_undistort_desc& u, const unsigned char* src, long long src_pitch, unsigned char* dst, long long dst_pitch)
{
    L3DUndistImage d;
    memset(&d, 0, sizeof(d));
    d.src = src; d.dst = dst; d.src_pitch = src_pitch; d.dst_pitch = dst_pitch;
    d.width = u.width; d.height = u.height; d.channels = u.channels;
    d.out_width = ud_out_width(u); d.out_height = ud_out_height(u);
    d.tiles_x = (d.out_width + UD_TW - 1) / UD_TW;
    const bool new_k = u.new_fx != 0.0 || u.new_fy != 0.0 || u.new_cx != 0.0 || u.new_cy != 0.0;
    const double nfx = new_k ? u.new_fx : u.fx, nfy = new_k ? u.new_fy : u.fy, ncx = new_k ? u.new_cx : u.cx, ncy = new_k ? u.new_cy : u.cy;
    const double det = nfx * nfy, id = 1.0 / det;
    d.ir0 = nfy * id; d.ir2 = -(ncx * nfy) * id; d.ir4 = nfx * id; d.ir5 = -(nfx * ncy) * id;
    d.fx = u.fx; d.fy = u.fy; d.cx = u.cx; d.cy = u.cy;
    if (u.model == L3D_LENS_FISHEYE) {
        d.kind = UD_FISHEYE;
        d.k1 = u.fisheye[0]; d.k2 = u.fisheye[1]; d.k3 = u.fisheye[2]; d.k4 = u.fisheye[3];
        return d;
    }
    d.k1 = u.radial[0]; d.k2 = u.radial[1]; d.k3 = u.radial[2]; d.p1 = u.tangential[0]; d.p2 = u.tangential[1];
    d.k4 = u.rational[0]; d.k5 = u.rational[1]; d.k6 = u.rational[2];
    d.full_radial = d.k2 != 0.0 || d.k3 != 0.0;
    d.tangential = d.p1 != 0.0 || d.p2 != 0.0;
    d.kind = d.k4 != 0.0 || d.k5 != 0.0 || d.k6 != 0.0 ? UD_RATIONAL : UD_RADTAN;
    return d;
}

// The column tables of the fisheye images among imgs[0, n): x_0 = ir2, x_{j+1} = x_j + ir0, summed in order as OpenCV's loop does.
// Images whose (ir0, ir2) agree share one table (its prefixes are the same), as long as the widest output among them.  Sets every fisheye
// image's xcol; the tables are uploaded on the context's stream.
static int ud_column_tables(l3d_ctx* c, UndistortState& s, L3DUndistImage* imgs, int n)
{
    struct Key { double ir0, ir2; int width; size_t off; };
    std::vector<Key> keys;
    std::vector<int> which(n, -1);
    for (int i = 0; i < n; ++i) {
        if (imgs[i].kind != UD_FISHEYE) continue;
        size_t k = 0;
        while (k < keys.size() && !(keys[k].ir0 == imgs[i].ir0 && keys[k].ir2 == imgs[i].ir2)) ++k;
        if (k == keys.size()) keys.push_back(Key{imgs[i].ir0, imgs[i].ir2, 0, 0});
        keys[k].width = std::max(keys[k].width, imgs[i].out_width);
        which[i] = (int)k;
    }
    if (keys.empty()) return L3D_OK;
    size_t total = 0;
    for (Key& k : keys) { k.off = total; total += (size_t)k.width; }
    s.h_cols.resize(total);
    for (const Key& k : keys) {
        double x = k.ir2;
        for (int j = 0; j < k.width; ++j) { s.h_cols[k.off + j] = x; x = x + k.ir0; }
    }
    int rc;
    L3D_RESERVE(s.d_cols, sizeof(double) * total, "fisheye column tables");
    // pageable host memory: staged before the call returns, like the descriptors
    L3D_CUDA(c, cudaMemcpyAsync(s.d_cols.p, s.h_cols.data(), sizeof(double) * total, cudaMemcpyHostToDevice, c->stream), "upload column tables");
    for (int i = 0; i < n; ++i)
        if (which[i] >= 0) imgs[i].xcol = (const double*)s.d_cols.p + keys[which[i]].off;
    return L3D_OK;
}

// one CTA row per output row, UD_TW output columns per CTA
static dim3 ud_grid(const l3d_undistort_desc& u) { return dim3((unsigned)((ud_out_width(u) + UD_TW - 1) / UD_TW), (unsigned)ud_out_height(u)); }

extern "C" {

int l3d_undistort_u8(l3d_ctx* c, int n, const l3d_undistort_desc* descs, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (n < 0 || (n && !descs)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_undistort_u8: bad arguments");
    for (int i = 0; i < n; ++i) {
        int rc = ud_check(c, descs[i], true, true, "l3d_undistort_u8");
        if (rc) return rc;
    }
    if (n == 0) return L3D_OK;
    cudaSetDevice(c->device);
    UndistortState& s = c->undist;
    int rc;
    std::vector<HostBlock> in, out;         // host mode: every source and output
    if (!on_device) {
        for (int i = 0; i < n; ++i) {
            const l3d_undistort_desc& u = descs[i];
            in.push_back({u.src, (size_t)u.src_pitch, (size_t)u.width * u.channels, (size_t)u.height});
            out.push_back({u.dst, (size_t)u.dst_pitch, (size_t)ud_out_width(u) * u.channels, (size_t)ud_out_height(u)});
        }
        if ((rc = l3d_stage_host(c, in.data(), n, out.data(), n))) return rc;
    }
    s.h_imgs.resize(n);
    for (int i = 0; i < n; ++i) {
        const l3d_undistort_desc& u = descs[i];
        if (on_device) s.h_imgs[i] = ud_image(u, u.src, u.src_pitch, u.dst, u.dst_pitch);
        else s.h_imgs[i] = ud_image(u, (const unsigned char*)in[i].dev, (long long)in[i].row_bytes, (unsigned char*)out[i].dev, (long long)out[i].row_bytes);
    }
    // the images grouped by lens kind: one grid per kind, each numbering its tiles from 0
    std::stable_sort(s.h_imgs.begin(), s.h_imgs.end(), [](const L3DUndistImage& a, const L3DUndistImage& b) { return a.kind < b.kind; });
    long long tiles[UD_KINDS] = {};
    int first[UD_KINDS + 1] = {};
    for (int i = 0; i < n; ++i) {
        L3DUndistImage& d = s.h_imgs[i];
        d.tile0 = tiles[d.kind];
        tiles[d.kind] += (long long)d.tiles_x * ((d.out_height + UD_TH - 1) / UD_TH);
        if (tiles[d.kind] >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_undistort_u8: more than 2^31 tiles in one call");
        first[d.kind + 1] = i + 1;
    }
    for (int k = 1; k <= UD_KINDS; ++k) first[k] = std::max(first[k], first[k - 1]);
    if ((rc = ud_column_tables(c, s, s.h_imgs.data(), n))) return rc;
    L3D_RESERVE(s.d_imgs, sizeof(L3DUndistImage) * (size_t)n, "undistort descriptors");
    // pageable host memory: the copy is staged before the call returns, so h_imgs may be rewritten by the next call right away
    L3D_CUDA(c, cudaMemcpyAsync(s.d_imgs.p, s.h_imgs.data(), sizeof(L3DUndistImage) * n, cudaMemcpyHostToDevice, c->stream), "upload descriptors");
    const L3DUndistImage* d_imgs = (const L3DUndistImage*)s.d_imgs.p;
    void (*const kernels[UD_KINDS])(const L3DUndistImage*, int) = {k_undistort_u8<UD_RADTAN>, k_undistort_u8<UD_RATIONAL>, k_undistort_u8<UD_FISHEYE>};
    for (int k = 0; k < UD_KINDS; ++k) {
        if (first[k + 1] == first[k]) continue;
        kernels[k]<<<(unsigned int)tiles[k], UD_TW, 0, c->stream>>>(d_imgs + first[k], first[k + 1] - first[k]);
        ++c->launches;
        L3D_CUDA(c, cudaGetLastError(), "k_undistort_u8");
    }
    if (!on_device && (rc = l3d_unstage_host(c, out.data(), n, "l3d_undistort_u8"))) return rc;
    return L3D_OK;
}

int l3d_undistort_map(l3d_ctx* c, const l3d_undistort_desc* desc, int16_t* map_xy, uint16_t* map_frac, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (!desc || !map_xy || !map_frac) return l3d_fail(c, L3D_ERR_INVALID, "l3d_undistort_map: null pointer");
    if (on_device && (((uintptr_t)map_xy & 3) || ((uintptr_t)map_frac & 1))) return l3d_fail(c, L3D_ERR_INVALID, "l3d_undistort_map: misaligned map");
    int rc = ud_check(c, *desc, false, true, "l3d_undistort_map");
    if (rc) return rc;
    cudaSetDevice(c->device);
    const size_t px = (size_t)ud_out_width(*desc) * ud_out_height(*desc);
    short2* xy = (short2*)map_xy; unsigned short* fr = map_frac;
    HostBlock out[2] = {host_array(map_xy, 4 * px), host_array(map_frac, 2 * px)};
    if (!on_device) {
        if ((rc = l3d_stage_host(c, nullptr, 0, out, 2))) return rc;
        xy = (short2*)out[0].dev; fr = (unsigned short*)out[1].dev;
    }
    L3DUndistImage d = ud_image(*desc, nullptr, 0, nullptr, 0);
    if ((rc = ud_column_tables(c, c->undist, &d, 1))) return rc;
    void (*const kernels[UD_KINDS])(L3DUndistImage, short2*, unsigned short*) = {k_undistort_map<UD_RADTAN>, k_undistort_map<UD_RATIONAL>,
                                                                                 k_undistort_map<UD_FISHEYE>};
    kernels[d.kind]<<<ud_grid(*desc), UD_TW, 0, c->stream>>>(d, xy, fr);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_undistort_map");
    if (!on_device && (rc = l3d_unstage_host(c, out, 2, "l3d_undistort_map"))) return rc;
    return L3D_OK;
}

int l3d_remap_u8(l3d_ctx* c, const l3d_undistort_desc* desc, const int16_t* map_xy, const uint16_t* map_frac, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (!desc || !map_xy || !map_frac) return l3d_fail(c, L3D_ERR_INVALID, "l3d_remap_u8: null pointer");
    if (on_device && (((uintptr_t)map_xy & 3) || ((uintptr_t)map_frac & 1))) return l3d_fail(c, L3D_ERR_INVALID, "l3d_remap_u8: misaligned map");
    int rc = ud_check(c, *desc, true, false, "l3d_remap_u8");
    if (rc) return rc;
    cudaSetDevice(c->device);
    const l3d_undistort_desc& u = *desc;
    const size_t px = (size_t)ud_out_width(u) * ud_out_height(u), row = (size_t)u.width * u.channels, out_row = (size_t)ud_out_width(u) * u.channels;
    L3DUndistImage d = ud_image(u, u.src, u.src_pitch, u.dst, u.dst_pitch);
    const short2* xy = (const short2*)map_xy; const unsigned short* fr = map_frac;
    HostBlock out[1] = {{u.dst, (size_t)u.dst_pitch, out_row, (size_t)ud_out_height(u)}};
    if (!on_device) {
        HostBlock in[3] = {{u.src, (size_t)u.src_pitch, row, (size_t)u.height}, host_array(map_xy, 4 * px), host_array(map_frac, 2 * px)};
        if ((rc = l3d_stage_host(c, in, 3, out, 1))) return rc;
        d.src = (const unsigned char*)in[0].dev; d.dst = (unsigned char*)out[0].dev; d.src_pitch = (long long)row; d.dst_pitch = (long long)out_row;
        xy = (const short2*)in[1].dev; fr = (const unsigned short*)in[2].dev;
    }
    if (u.channels == 3) k_remap_u8<3><<<ud_grid(u), UD_TW, 0, c->stream>>>(d, xy, fr);
    else k_remap_u8<1><<<ud_grid(u), UD_TW, 0, c->stream>>>(d, xy, fr);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_remap_u8");
    if (!on_device && (rc = l3d_unstage_host(c, out, 1, "l3d_remap_u8"))) return rc;
    return L3D_OK;
}

int l3d_undistort_points(l3d_ctx* c, int n, const l3d_points_desc* sets, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (n < 0 || (n && !sets)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_undistort_points: bad arguments");
    char buf[160];
    long long total = 0;
    for (int i = 0; i < n; ++i) {
        const l3d_points_desc& d = sets[i];
        int rc = ud_check_camera(c, d.cam, "l3d_undistort_points");
        if (rc) return rc;
        if (d.count < 0 || (d.count > 0 && (!d.src || !d.dst))) {
            snprintf(buf, sizeof(buf), "l3d_undistort_points: set %d: %s", i, d.count < 0 ? "count < 0" : "null point pointer");
            return l3d_fail(c, L3D_ERR_INVALID, buf);
        }
        if (d.count > (1ll << 38) - total) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_undistort_points: more than 2^38 points in one call");
        total += d.count;
    }
    if (total == 0) return L3D_OK;
    cudaSetDevice(c->device);
    UndistortState& s = c->undist;
    int rc;
    std::vector<HostBlock> in, out;         // host mode: the points of every non-empty set
    if (!on_device) {
        for (int i = 0; i < n; ++i)
            if (sets[i].count) {
                in.push_back(host_array(sets[i].src, 8 * (size_t)sets[i].count));
                out.push_back(host_array(sets[i].dst, 8 * (size_t)sets[i].count));
            }
        if ((rc = l3d_stage_host(c, in.data(), (int)in.size(), out.data(), (int)out.size()))) return rc;
    }
    // the non-empty sets only: every point then lies in the set the search over p0 finds
    s.h_sets.clear();
    long long p0 = 0;
    for (int i = 0; i < n; ++i) {
        const l3d_points_desc& d = sets[i];
        if (!d.count) continue;
        const size_t j = s.h_sets.size();
        s.h_sets.push_back(on_device ? up_set(d.cam, d.src, d.dst, p0) : up_set(d.cam, (const float*)in[j].dev, (float*)out[j].dev, p0));
        p0 += d.count;
    }
    const int m = (int)s.h_sets.size();
    L3D_RESERVE(s.d_sets, sizeof(L3DPointSet) * (size_t)m, "point set descriptors");
    // pageable host memory: the copy is staged before the call returns, so h_sets may be rewritten by the next call right away
    L3D_CUDA(c, cudaMemcpyAsync(s.d_sets.p, s.h_sets.data(), sizeof(L3DPointSet) * m, cudaMemcpyHostToDevice, c->stream), "upload point sets");
    k_undistort_points<<<(unsigned int)((total + UP_THREADS - 1) / UP_THREADS), UP_THREADS, 0, c->stream>>>((const L3DPointSet*)s.d_sets.p, m, total);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_undistort_points");
    if (!on_device && (rc = l3d_unstage_host(c, out.data(), (int)out.size(), "l3d_undistort_points"))) return rc;
    return L3D_OK;
}

} // extern "C"
