// line3d_newk.cc — the two new-camera-matrix functions of OpenCV that go with Line3D::undistortImage(..., newK, out_width, out_height):
// cv::getOptimalNewCameraMatrix (radtan lenses) and cv::fisheye::estimateNewCameraMatrixForUndistortRectify, restated in double on
// the host step for step as OpenCV 4.13 computes them (DESIGN.md §4a).  They touch a few dozen points, so there is no kernel.
// Skew is taken as zero, as in the undistortion itself.
#include "../../include/line3d.h"
#include "../../include/l3dpp_capi.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <climits>
#include <stdexcept>
#include <string>

namespace L3DPP {

namespace {

struct Pt { double x, y; };

void check_camera(const Matrix3d& K, int width, int height, const char* what)
{
    if (width < 1 || height < 1) throw std::invalid_argument(std::string(what) + ": the image size must be at least 1 x 1");
    if (!std::isfinite(K(0, 0)) || !std::isfinite(K(1, 1)) || K(0, 0) == 0.0 || K(1, 1) == 0.0)
        throw std::invalid_argument(std::string(what) + ": fx and fy must be finite and non-zero");
}

// cv::undistortPoints(src, dst, K, D, R = I, P) with its default criterion: 5 iterations of the fixed-point step, no tolerance test
// (cv2 4.13 matches 5 exactly and no other count).  D = (k1, k2, p1, p2, k3, k4, k5, k6); the thin-prism terms are zero.  P: the
// new camera matrix, or null for normalised coordinates.
Pt undistort_point_radtan(Pt p, const Matrix3d& K, const double k[8], const Matrix3d* P)
{
    const double fx = K(0, 0), fy = K(1, 1), cx = K(0, 2), cy = K(1, 2), ifx = 1. / fx, ify = 1. / fy;
    double x = (p.x - cx) * ifx, y = (p.y - cy) * ify;
    const double x0 = x, y0 = y;
    for (int j = 0; j < 5; ++j) {
        const double r2 = x * x + y * y;
        const double icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
        if (icdist < 0) {   // OpenCV gives up on the point: its distorted normalised position
            x = (p.x - cx) * ifx;
            y = (p.y - cy) * ify;
            break;
        }
        const double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x);
        const double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y;
        x = (x0 - deltaX) * icdist;
        y = (y0 - deltaY) * icdist;
    }
    if (P) { x = (*P)(0, 0) * x + (*P)(0, 2); y = (*P)(1, 1) * y + (*P)(1, 2); }
    return Pt{x, y};
}

// OpenCV's getUndistortRectangles: a 9 x 9 grid over [0, w-1] x [0, h-1] (in double), undistorted; inner = the rectangle inside the
// undistorted border, outer = the bounding box of the 32 border points only (an interior point that a folding lens carries past the
// border does not widen it; cv2 4.13 agrees with this and not with the box of all 81).  Rectangles as x, y, width, height.
void undistort_rectangles(const Matrix3d& K, const double k[8], const Matrix3d* P, int w, int h, double inner[4], double outer[4])
{
    const int N = 9;
    double iX0 = -DBL_MAX, iX1 = DBL_MAX, iY0 = -DBL_MAX, iY1 = DBL_MAX;
    double oX0 = DBL_MAX, oX1 = -DBL_MAX, oY0 = DBL_MAX, oY1 = -DBL_MAX;
    for (int y = 0; y < N; ++y)
        for (int x = 0; x < N; ++x) {
            if (x != 0 && x != N - 1 && y != 0 && y != N - 1) continue;
            const Pt p = undistort_point_radtan(Pt{(double)x * (w - 1) / (N - 1), (double)y * (h - 1) / (N - 1)}, K, k, P);
            oX0 = std::min(oX0, p.x); oX1 = std::max(oX1, p.x); oY0 = std::min(oY0, p.y); oY1 = std::max(oY1, p.y);
            if (x == 0) iX0 = std::max(iX0, p.x);
            if (x == N - 1) iX1 = std::min(iX1, p.x);
            if (y == 0) iY0 = std::max(iY0, p.y);
            if (y == N - 1) iY1 = std::min(iY1, p.y);
        }
    inner[0] = iX0; inner[1] = iY0; inner[2] = iX1 - iX0; inner[3] = iY1 - iY0;
    outer[0] = oX0; outer[1] = oY0; outer[2] = oX1 - oX0; outer[3] = oY1 - oY0;
}

// an integer rounded from v by `round` (std::nearbyint: cvRound; std::ceil / std::floor: cvCeil / cvFloor), saturated to int
template <class F>
int sat_int(double v, F round)
{
    const double r = round(v);
    return r >= (double)INT_MAX ? INT_MAX : r <= (double)INT_MIN ? INT_MIN : r == r ? (int)r : 0;
}

// cv::Rect's r &= Rect(0, 0, w, h): the intersection, or an empty rectangle
void clip_rect(int r[4], int w, int h)
{
    const int x1 = std::max(r[0], 0), y1 = std::max(r[1], 0);
    const int rw = std::min(r[0] + r[2], w) - x1, rh = std::min(r[1] + r[3], h) - y1;
    if (rw <= 0 || rh <= 0) { r[0] = r[1] = r[2] = r[3] = 0; return; }
    r[0] = x1; r[1] = y1; r[2] = rw; r[3] = rh;
}

// cv::fisheye::undistortPoints(src, dst, K, D) with its default criterion (at most 10 Newton steps, stop when |step| < 1e-8):
// normalised coordinates, or (-1e6, -1e6) where OpenCV's iteration does not converge or theta changes sign
Pt undistort_point_fisheye(Pt p, const Matrix3d& K, const double k[4])
{
    const double pwx = (p.x - K(0, 2)) / K(0, 0), pwy = (p.y - K(1, 2)) / K(1, 1);
    double theta_d = std::sqrt(pwx * pwx + pwy * pwy);
    theta_d = std::min(std::max(-M_PI / 2., theta_d), M_PI / 2.);
    bool converged = false;
    double theta = theta_d, scale = 0.0;
    if (std::fabs(theta_d) > 1e-8) {
        for (int j = 0; j < 10; ++j) {
            const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2, theta8 = theta6 * theta2;
            const double k0_theta2 = k[0] * theta2, k1_theta4 = k[1] * theta4, k2_theta6 = k[2] * theta6, k3_theta8 = k[3] * theta8;
            const double theta_fix = (theta * (1 + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d) /
                                     (1 + 3 * k0_theta2 + 5 * k1_theta4 + 7 * k2_theta6 + 9 * k3_theta8);
            theta = theta - theta_fix;
            if (std::fabs(theta_fix) < 1e-8) { converged = true; break; }
        }
        scale = std::tan(theta) / theta_d;
    } else {
        converged = true;
    }
    const bool flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
    if (converged && !flipped) return Pt{pwx * scale, pwy * scale};
    return Pt{-1000000.0, -1000000.0};
}

Matrix3d camera(double fx, double fy, double cx, double cy)
{
    Matrix3d M;
    std::memset(&M, 0, sizeof(M));
    M(0, 0) = fx; M(1, 1) = fy; M(0, 2) = cx; M(1, 2) = cy; M(2, 2) = 1.0;
    return M;
}

}  // namespace

Matrix3d Line3D::getOptimalNewCameraMatrix(const Matrix3d& K, const LensDistortion& lens, int width, int height, double alpha, int new_width,
                                           int new_height, int validPixROI[4], bool centerPrincipalPoint)
{
    const char* what = "getOptimalNewCameraMatrix";
    check_camera(K, width, height, what);
    if (lens.model != LensDistortion::RADTAN) throw std::invalid_argument("getOptimalNewCameraMatrix: a radtan lens (fisheye: estimateNewCameraMatrixForUndistortRectify)");
    if (new_width < 0 || new_height < 0) throw std::invalid_argument("getOptimalNewCameraMatrix: a negative new size");
    const double k[8] = {lens.k[0], lens.k[1], lens.p[0], lens.p[1], lens.k[2], lens.k[3], lens.k[4], lens.k[5]};
    const Matrix3d A = camera(K(0, 0), K(1, 1), K(0, 2), K(1, 2));
    const int nw = (long long)new_width * new_height != 0 ? new_width : width, nh = (long long)new_width * new_height != 0 ? new_height : height;
    double inner[4], outer[4];
    Matrix3d M = A;
    int roi[4];
    if (centerPrincipalPoint) {
        const double cx0 = A(0, 2), cy0 = A(1, 2), cx = (nw - 1) * 0.5, cy = (nh - 1) * 0.5;
        undistort_rectangles(A, k, &A, width, height, inner, outer);
        const double s0 = std::max(std::max(std::max(cx / (cx0 - inner[0]), cy / (cy0 - inner[1])), cx / (inner[0] + inner[2] - cx0)),
                                   cy / (inner[1] + inner[3] - cy0));
        const double s1 = std::min(std::min(std::min(cx / (cx0 - outer[0]), cy / (cy0 - outer[1])), cx / (outer[0] + outer[2] - cx0)),
                                   cy / (outer[1] + outer[3] - cy0));
        const double s = s0 * (1 - alpha) + s1 * alpha;
        M(0, 0) *= s; M(1, 1) *= s; M(0, 2) = cx; M(1, 2) = cy;
        const auto ceil = [](double v) { return std::ceil(v); };
        const auto floor = [](double v) { return std::floor(v); };
        roi[0] = sat_int((inner[0] - cx0) * s + cx, ceil);
        roi[1] = sat_int((inner[1] - cy0) * s + cy, ceil);
        roi[2] = sat_int(inner[2] * s, floor);
        roi[3] = sat_int(inner[3] * s, floor);
    } else {
        undistort_rectangles(A, k, nullptr, width, height, inner, outer);   // in normalised coordinates
        const double fx0 = (nw - 1) / inner[2], fy0 = (nh - 1) / inner[3], cx0 = -fx0 * inner[0], cy0 = -fy0 * inner[1];
        const double fx1 = (nw - 1) / outer[2], fy1 = (nh - 1) / outer[3], cx1 = -fx1 * outer[0], cy1 = -fy1 * outer[1];
        M(0, 0) = fx0 * (1 - alpha) + fx1 * alpha;
        M(1, 1) = fy0 * (1 - alpha) + fy1 * alpha;
        M(0, 2) = cx0 * (1 - alpha) + cx1 * alpha;
        M(1, 2) = cy0 * (1 - alpha) + cy1 * alpha;
        undistort_rectangles(A, k, &M, width, height, inner, outer);
        for (int i = 0; i < 4; ++i) roi[i] = sat_int(inner[i], [](double v) { return std::nearbyint(v); });   // cv::Rect(Rect_<double>): cvRound
    }
    clip_rect(roi, nw, nh);
    if (validPixROI) std::memcpy(validPixROI, roi, sizeof(roi));
    return M;
}

Matrix3d Line3D::estimateNewCameraMatrixForUndistortRectify(const Matrix3d& K, const LensDistortion& lens, int width, int height, double balance,
                                                            int new_width, int new_height, double fov_scale)
{
    check_camera(K, width, height, "estimateNewCameraMatrixForUndistortRectify");
    if (lens.model != LensDistortion::FISHEYE) throw std::invalid_argument("estimateNewCameraMatrixForUndistortRectify: a fisheye lens");
    const int w = width, h = height;
    balance = std::min(std::max(balance, 0.0), 1.0);
    // the four edge midpoints (integer halves, as OpenCV forms them), undistorted to normalised coordinates
    Pt p[4] = {{(double)(w / 2), 0.0}, {(double)w, (double)(h / 2)}, {(double)(w / 2), (double)h}, {0.0, (double)(h / 2)}};
    for (Pt& q : p) q = undistort_point_fisheye(q, K, lens.k);
    double cn[2] = {(((p[0].x + p[1].x) + p[2].x) + p[3].x) * (1. / 4), (((p[0].y + p[1].y) + p[2].y) + p[3].y) * (1. / 4)};   // cv::mean
    const double aspect_ratio = K(0, 0) / K(1, 1);
    cn[1] *= aspect_ratio;
    for (Pt& q : p) q.y *= aspect_ratio;
    double minx = DBL_MAX, miny = DBL_MAX, maxx = -DBL_MAX, maxy = -DBL_MAX;
    for (const Pt& q : p) {
        miny = std::min(miny, q.y); maxy = std::max(maxy, q.y);
        minx = std::min(minx, q.x); maxx = std::max(maxx, q.x);
    }
    const double f1 = w * 0.5 / (cn[0] - minx), f2 = w * 0.5 / (maxx - cn[0]);
    const double f3 = h * 0.5 * aspect_ratio / (cn[1] - miny), f4 = h * 0.5 * aspect_ratio / (maxy - cn[1]);
    const double fmin = std::min(f1, std::min(f2, std::min(f3, f4))), fmax = std::max(f1, std::max(f2, std::max(f3, f4)));
    double f = balance * fmin + (1.0 - balance) * fmax;
    f *= fov_scale > 0 ? 1.0 / fov_scale : 1.0;
    double new_f[2] = {f, f}, new_c[2] = {-cn[0] * f + w * 0.5, -cn[1] * f + h * aspect_ratio * 0.5};
    new_f[1] /= aspect_ratio;
    new_c[1] /= aspect_ratio;
    if (new_width > 0 && new_height > 0) {   // !Size::empty()
        const double rx = new_width / (double)width, ry = new_height / (double)height;
        new_f[0] *= rx; new_f[1] *= ry;
        new_c[0] *= rx; new_c[1] *= ry;
    }
    return camera(new_f[0], new_f[1], new_c[0], new_c[1]);
}

}  // namespace L3DPP

// ================================================================================================ C wrapper (include/l3dpp_capi.h)
using namespace L3DPP;

static LensDistortion lens_from9(const double* lens9)
{
    LensDistortion lens;
    lens.model = (int)lens9[0];
    for (int k = 0; k < 6; ++k) lens.k[k] = lens9[1 + k];
    lens.p[0] = lens9[7]; lens.p[1] = lens9[8];
    return lens;
}

extern "C" {
int l3dpp_optimal_new_camera_matrix(const double* K, const double* lens9, int width, int height, double alpha, int new_width, int new_height,
                                    int center_principal_point, double* newK, int* roi)
{
    Matrix3d Km;
    std::memcpy(Km.m, K, 72);
    try {
        const Matrix3d M = Line3D::getOptimalNewCameraMatrix(Km, lens_from9(lens9), width, height, alpha, new_width, new_height, roi,
                                                             center_principal_point != 0);
        std::memcpy(newK, M.m, 72);
    } catch (const std::invalid_argument&) { return -1; }
    return 0;
}
int l3dpp_fisheye_new_camera_matrix(const double* K, const double* lens9, int width, int height, double balance, int new_width, int new_height,
                                    double fov_scale, double* newK)
{
    Matrix3d Km;
    std::memcpy(Km.m, K, 72);
    try {
        const Matrix3d M = Line3D::estimateNewCameraMatrixForUndistortRectify(Km, lens_from9(lens9), width, height, balance, new_width, new_height,
                                                                              fov_scale);
        std::memcpy(newK, M.m, 72);
    } catch (const std::invalid_argument&) { return -1; }
    return 0;
}
}
