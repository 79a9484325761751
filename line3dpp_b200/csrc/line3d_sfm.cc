// line3d_sfm.cc — the input side of the reference's six frontends as library readers: NVM (main_vsfm.cpp:143-310), Bundler
// (main_bundler.cpp:143-286), COLMAP text and binary (main_colmap.cpp:140-401), mavmap (main_mavmap.cpp:153-321), OpenMVG
// (main_openmvg.cpp:136-410) and Pix4D (main_pix4d.cpp:163-420); the static helpers only these frontends use (Line3D::rotationFromQ,
// rotationFromRPY, decomposeProjectionMatrix); and their C wrappers.  Host code; the Pix4D reader triangulates its tie points and
// computes the median depths through the C ABI (l3d_triangulate_points, l3d_median_depths).  The file needs no CUDA header, so it
// builds alone (with stand-ins for those two entries) for the sanitizer test.
//
// Every reader takes input from outside the program: a malformed file returns false with *error naming the file and the problem
// (the line or JSON path where the format has them); nothing is allocated beyond what the bytes read justify, whatever count a header
// claims; JSON nesting is capped at JSON_MAX_DEPTH.
#include "../../include/line3d_io.h"
#include "../../include/l3d_capi.h"
#include "../../include/l3dpp_capi.h"
#include "l3dpp_wrap.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <map>
#include <sstream>

namespace L3DPP {

// ------------------------------------------------------------------------------------------------ camera algebra
// Every product sums left to right.  The negations come after the sums: -(a + b) is -0 where (-a) + (-b) is +0, so the two spellings
// are not interchangeable when a component cancels exactly.
static Matrix3d zero3() { Matrix3d m; std::memset(m.m, 0, sizeof(m.m)); return m; }
static Vector3d neg(const Vector3d& v) { return Vector3d(-v.x, -v.y, -v.z); }
static Vector3d mul(const Matrix3d& R, const Vector3d& v)
{
    return Vector3d(R(0, 0) * v.x + R(0, 1) * v.y + R(0, 2) * v.z, R(1, 0) * v.x + R(1, 1) * v.y + R(1, 2) * v.z,
                    R(2, 0) * v.x + R(2, 1) * v.y + R(2, 2) * v.z);
}
static Vector3d mul_transposed(const Matrix3d& R, const Vector3d& v)      // R^T v
{
    return Vector3d(R(0, 0) * v.x + R(1, 0) * v.y + R(2, 0) * v.z, R(0, 1) * v.x + R(1, 1) * v.y + R(2, 1) * v.z,
                    R(0, 2) * v.x + R(1, 2) * v.y + R(2, 2) * v.z);
}
static Vector3d translation_of(const Matrix3d& R, const Vector3d& C) { return neg(mul(R, C)); }           // t = -R C
static Vector3d center_of(const Matrix3d& R, const Vector3d& t) { return neg(mul_transposed(R, t)); }    // C = -R^T t

// |C - X| rounded to float: the reference keeps depths in float vectors (main_vsfm.cpp:228, main_colmap.cpp:386-401)
static float point_depth(const Vector3d& C, const Vector3d& X)
{
    const double dx = C.x - X.x, dy = C.y - X.y, dz = C.z - X.z;
    return (float)std::sqrt(dx * dx + dy * dy + dz * dz);
}

// element size/2 of the sorted depths; 0 for none
static float median_of(std::vector<float>& d)
{
    if (d.empty()) return 0.0f;
    std::sort(d.begin(), d.end());
    return d[d.size() / 2];
}

// ------------------------------------------------------------------------------------------------ helpers on Line3D
// the rotation of a unit quaternion (line3D.cc:2737-2754 after its normalisation; main_vsfm.cpp:193-203 uses it as stored)
static Matrix3d quaternion_matrix(double w, double x, double y, double z)
{
    Matrix3d R;
    R(0, 0) = 1.0 - 2.0 * y * y - 2.0 * z * z; R(0, 1) = 2.0 * x * y - 2.0 * z * w; R(0, 2) = 2.0 * x * z + 2.0 * y * w;
    R(1, 0) = 2.0 * x * y + 2.0 * z * w; R(1, 1) = 1.0 - 2.0 * x * x - 2.0 * z * z; R(1, 2) = 2.0 * y * z - 2.0 * x * w;
    R(2, 0) = 2.0 * x * z - 2.0 * y * w; R(2, 1) = 2.0 * y * z + 2.0 * x * w; R(2, 2) = 1.0 - 2.0 * x * x - 2.0 * y * y;
    return R;
}

Matrix3d Line3D::rotationFromQ(const double Qw, const double Qx, const double Qy, const double Qz)   // line3D.cc:2737-2754
{
    const double n = std::sqrt(Qw * Qw + Qx * Qx + Qy * Qy + Qz * Qz);
    return quaternion_matrix(Qw / n, Qx / n, Qy / n, Qz / n);
}

// Eigen's AngleAxisd(angle, axis).toRotationMatrix() for a unit axis e_k: the diagonal entry of the axis is (1 - c) + c
static Matrix3d axis_rotation(double angle, int k)
{
    const double s = std::sin(angle), c = std::cos(angle);
    Matrix3d R = zero3();
    const int i = (k + 1) % 3, j = (k + 2) % 3;
    R(k, k) = (1.0 - c) + c;
    R(i, i) = c; R(j, j) = c;
    R(i, j) = -s; R(j, i) = s;
    return R;
}

static Matrix3d mul(const Matrix3d& a, const Matrix3d& b)      // inner dimension summed left to right
{
    Matrix3d m;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) m(r, c) = a(r, 0) * b(0, c) + a(r, 1) * b(1, c) + a(r, 2) * b(2, c);
    return m;
}

Matrix3d Line3D::rotationFromRPY(const double roll, const double pitch, const double yaw)      // line3D.cc:2714-2727
{
    return mul(mul(axis_rotation(yaw, 2), axis_rotation(pitch, 1)), axis_rotation(roll, 0));
}

// line3D.cc:2784-2852: RQ decomposition of P's left 3x3 block by three Givens rotations (Hartley & Zisserman), in the reference's order
void Line3D::decomposeProjectionMatrix(const double P[12], Matrix3d& K, Matrix3d& R, Vector3d& t)
{
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) K(r, c) = P[4 * r + c];
    auto givens = [](int a, int b, double s, double c) {      // identity with c at (a,a), (b,b); -s at (a,b); s at (b,a)
        Matrix3d G = zero3();
        G(3 - a - b, 3 - a - b) = 1.0;
        G(a, a) = c; G(b, b) = c; G(a, b) = -s; G(b, a) = s;
        return G;
    };
    double h = std::sqrt(K(2, 1) * K(2, 1) + K(2, 2) * K(2, 2));
    const Matrix3d Rx = givens(1, 2, K(2, 1) / h, -K(2, 2) / h);
    K = mul(K, Rx);
    h = std::sqrt(K(2, 0) * K(2, 0) + K(2, 2) * K(2, 2));
    const Matrix3d Ry = givens(0, 2, K(2, 0) / h, -K(2, 2) / h);
    K = mul(K, Ry);
    h = std::sqrt(K(1, 0) * K(1, 0) + K(1, 1) * K(1, 1));
    const Matrix3d Rz = givens(0, 1, K(1, 0) / h, -K(1, 1) / h);
    K = mul(K, Rz);
    Matrix3d Sign = zero3();
    for (int i = 0; i < 3; ++i) Sign(i, i) = K(i, i) < 0 ? -1.0 : 1.0;
    K = mul(K, Sign);                                      // change the sign of columns
    const Matrix3d Rt = mul(mul(mul(Rx, Ry), Rz), Sign);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R(r, c) = Rt(c, r);
    // t = K^-1 P4 with the inverse as Eigen forms a 3x3 one: cofactors of column 0, det, every cofactor times 1/det
    auto cof = [&K](int i, int j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        return K(i1, j1) * K(i2, j2) - K(i1, j2) * K(i2, j1);
    };
    const double det = (cof(0, 0) * K(0, 0) + cof(1, 0) * K(1, 0)) + cof(2, 0) * K(2, 0), invdet = 1.0 / det;
    Matrix3d Ki;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) Ki(r, c) = cof(c, r) * invdet;
    t = mul(Ki, Vector3d(P[3], P[7], P[11]));
    const double n = 1.0 / K(2, 2);                        // normalise so that K(2,2) = 1
    for (int i = 0; i < 9; ++i) K.m[i] *= n;
}

std::list<unsigned int> sequentialNeighbors(unsigned int i, unsigned int n_cams, unsigned int num_neighbors)     // main_mavmap.cpp:312-321
{
    std::list<unsigned int> nb;
    const size_t n_before = num_neighbors / 2;
    for (long long j = (long long)i - 1; j >= 0 && nb.size() < n_before; --j) nb.push_back((unsigned int)j);
    for (long long j = (long long)i + 1; j < (long long)n_cams && nb.size() < num_neighbors; ++j) nb.push_back((unsigned int)j);
    return nb;
}

Matrix3d intrinsicsFromFocal(float focal, int w, int h)
{
    Matrix3d K = zero3();
    K(0, 0) = focal; K(1, 1) = focal; K(0, 2) = float(w) / 2.0f; K(1, 2) = float(h) / 2.0f; K(2, 2) = 1.0;
    return K;
}

// ------------------------------------------------------------------------------------------------ shared parsing helpers
static bool fail(std::string* error, const std::string& msg) { if (error) error->assign(msg); return false; }

// the whole token must be a number (strtod: correctly rounded, like the reference's stream extraction)
static bool to_double(const std::string& tok, double& v)
{
    if (tok.empty() || std::isspace((unsigned char)tok[0])) return false;
    char* end = nullptr;
    v = std::strtod(tok.c_str(), &end);
    return end == tok.c_str() + tok.size();
}

// n numbers from the whitespace-separated tokens of a line (further tokens are ignored, as the reference's stream reads ignore them)
static bool read_numbers(const std::string& line, double* out, int n)
{
    std::istringstream s(line);
    std::string tok;
    for (int i = 0; i < n; ++i)
        if (!(s >> tok) || !to_double(tok, out[i])) return false;
    return true;
}

// a camera's K, the radial / tangential distortion the frontend undistorts with and (COLMAP only) its full lens
struct Intrinsics { Matrix3d K; double radial[3], tangential[2]; LensDistortion lens; };

static SfMCamera empty_camera(unsigned int id)
{
    SfMCamera c;
    c.id = id; c.has_K = true; c.K = zero3(); c.focal = 0.0f; c.R = zero3(); c.median_depth = 0.0f;
    c.radial[0] = c.radial[1] = c.radial[2] = 0.0; c.tangential[0] = c.tangential[1] = 0.0;
    return c;
}

// ------------------------------------------------------------------------------------------------ NVM
// the view list "n  cam feature x y  ..." of point i at X in an NVM or Bundler file: each camera it names gets the point and its depth;
// false when the list is cut short or names a camera that does not exist
template <class Cam> static bool add_views(std::istream& s, unsigned int i, const Vector3d& X, std::vector<Cam>& cams, std::vector<std::vector<float> >& depths)
{
    unsigned int nviews = 0;
    s >> nviews;
    for (unsigned int j = 0; j < nviews; ++j) {
        unsigned int cam = 0, sift = 0; float x, y;
        s >> cam >> sift >> x >> y;
        if (!s || cam >= cams.size()) return false;
        cams[cam].worldpoints.push_back(i);
        depths[cam].push_back(point_depth(cams[cam].C, X));
    }
    return true;
}

bool readNVM(const std::string& path, std::vector<NVMCamera>& cams, std::string* error)
{
    cams.clear();
    std::ifstream f(path.c_str());
    if (!f) return fail(error, "cannot open " + path);
    std::string line;
    std::getline(f, line);                       // "NVM_V3"
    std::getline(f, line);                       // empty
    std::getline(f, line);
    unsigned int num_cams = 0;
    { std::stringstream s(line); s >> num_cams; }
    if (num_cams == 0) return fail(error, "No aligned cameras in NVM file!");     // main_vsfm.cpp:157-161
    for (unsigned int i = 0; i < num_cams; ++i) {   // appended as read: a count the file does not hold allocates nothing
        // a truncated or malformed camera line must not become a default camera (the reference has the same hole, main_vsfm.cpp:168-190)
        if (!std::getline(f, line)) return fail(error, "unexpected end of file in the camera list of " + path + " (camera " + std::to_string(i) + ")");
        std::stringstream s(line);
        NVMCamera c;
        double focal = 0, qw = 1, qx = 0, qy = 0, qz = 0, Cx = 0, Cy = 0, Cz = 0, dist = 0;
        if (!(s >> c.image >> focal >> qw >> qx >> qy >> qz >> Cx >> Cy >> Cz >> dist)) return fail(error, "malformed camera line " + std::to_string(i) + " in " + path);
        c.focal = (float)focal; c.distortion = (float)dist;
        c.R = quaternion_matrix(qw, qx, qy, qz);   // main_vsfm.cpp:193-203 (the quaternion is used as stored, not re-normalised)
        c.C = Vector3d(Cx, Cy, Cz);
        c.t = translation_of(c.R, c.C);
        c.median_depth = 0.0f;
        cams.push_back(c);
    }
    std::getline(f, line);                       // empty
    std::getline(f, line);
    unsigned int num_points = 0;
    { std::stringstream s(line); s >> num_points; }
    std::vector<std::vector<float> > depths(cams.size());
    for (unsigned int i = 0; i < num_points; ++i) {
        if (!std::getline(f, line)) break;
        std::istringstream s(line);
        double px = 0, py = 0, pz = 0, cr, cg, cb;
        s >> px >> py >> pz >> cr >> cg >> cb;
        if (!add_views(s, i, Vector3d(px, py, pz), cams, depths)) return fail(error, "malformed measurement list in " + path);
    }
    for (size_t i = 0; i < cams.size(); ++i) cams[i].median_depth = median_of(depths[i]);     // main_vsfm.cpp:301-303
    return true;
}

// ------------------------------------------------------------------------------------------------ Bundler
bool readBundler(const std::string& bundle_file, const std::string& image_list_file, std::vector<SfMCamera>& cams, std::string* error)
{
    cams.clear();
    std::ifstream f(bundle_file.c_str());
    if (!f) return fail(error, "cannot open " + bundle_file);
    std::string line;
    std::getline(f, line);                       // "# Bundle file v0.3"
    std::getline(f, line);
    unsigned int num_cams = 0, num_points = 0;
    { std::stringstream s(line); s >> num_cams >> num_points; }
    if (num_cams == 0 || num_points == 0) return fail(error, "No cameras and/or points in bundle file!");   // main_bundler.cpp:159-163
    for (unsigned int i = 0; i < num_cams; ++i) {   // appended as read, like the NVM cameras
        SfMCamera c = empty_camera(i);
        c.has_K = false;
        double focal = 0, d1 = 0, d2 = 0;
        bool good = (bool)std::getline(f, line);
        if (good) { std::stringstream s(line); good = (bool)(s >> focal >> d1 >> d2); }
        c.focal = (float)focal;
        c.radial[0] = (float)d1; c.radial[1] = (float)d2;                                                               // float pair, main_bundler.cpp:170, 183
        for (int j = 0; j < 3 && good; ++j) { good = (bool)std::getline(f, line); std::stringstream s(line); good = good && (bool)(s >> c.R(j, 0) >> c.R(j, 1) >> c.R(j, 2)); }
        for (int k = 0; k < 3; ++k) { c.R(1, k) *= -1.0; c.R(2, k) *= -1.0; }                                           // main_bundler.cpp:196-198
        good = good && (bool)std::getline(f, line);
        if (good) { std::stringstream s(line); good = (bool)(s >> c.t.x >> c.t.y >> c.t.z); }
        if (!good) return fail(error, "truncated or malformed camera " + std::to_string(i) + " in " + bundle_file);
        c.t.y *= -1.0; c.t.z *= -1.0;                                                                                    // main_bundler.cpp:210-212
        c.C = center_of(c.R, c.t);
        cams.push_back(c);
    }
    std::vector<std::vector<float> > depths(cams.size());
    for (unsigned int i = 0; i < num_points; ++i) {
        if (!std::getline(f, line)) break;
        double px = 0, py = 0, pz = 0;
        { std::istringstream s(line); s >> px >> py >> pz; }
        std::getline(f, line);                   // colour
        std::getline(f, line);                   // view list
        std::istringstream s(line);
        if (!add_views(s, i, Vector3d(px, py, pz), cams, depths)) return fail(error, "malformed view list in " + bundle_file);
    }
    for (size_t i = 0; i < cams.size(); ++i) cams[i].median_depth = median_of(depths[i]);
    if (!image_list_file.empty()) {              // main_bundler.cpp:264-286: the first token of line i names image i
        std::ifstream l(image_list_file.c_str());
        size_t id = 0;
        while (std::getline(l, line)) {
            std::stringstream s(line);
            std::string fname;
            s >> fname;
            if (!fname.empty() && id < cams.size()) cams[id].image = fname;
            ++id;
        }
    }
    return true;
}

// ------------------------------------------------------------------------------------------------ COLMAP
// COLMAP's camera models (colmap/sensor/models.h): name, model_id, number of parameters.  `lens` 0: not undistortable here (rejected),
// 1: radtan, 2: fisheye.
struct ColmapModel { const char* name; int id, num_params, lens; };
static const ColmapModel kColmapModels[] = {
    {"SIMPLE_PINHOLE", 0, 3, 1}, {"PINHOLE", 1, 4, 1}, {"SIMPLE_RADIAL", 2, 4, 1}, {"RADIAL", 3, 5, 1}, {"OPENCV", 4, 8, 1},
    {"OPENCV_FISHEYE", 5, 8, 2}, {"FULL_OPENCV", 6, 12, 1}, {"FOV", 7, 5, 0}, {"SIMPLE_RADIAL_FISHEYE", 8, 4, 2}, {"RADIAL_FISHEYE", 9, 5, 2},
    {"THIN_PRISM_FISHEYE", 10, 12, 0}, {"RAD_TAN_THIN_PRISM_FISHEYE", 11, 16, 0},
};


// K, the radial / tangential pair of main_colmap.cpp:160-234 and the full lens of one camera from its parameters in COLMAP's order
static bool colmap_intrinsics(const ColmapModel* m, const std::string& model, unsigned int cam, const double* q, bool want_lens, Intrinsics& in,
                              std::string* error)
{
    if (!m || m->lens == 0) return fail(error, "camera model " + model + " unknown! (camera " + std::to_string(cam) + ")");
    if (m->lens == 2 && !want_lens)
        return fail(error, "camera " + std::to_string(cam) + " uses the fisheye model " + model + ": its distortion has no place in radial / tangential, "
                           "read the model with the lenses argument of readColmap");
    double fx = 0, fy = 0, cx = 0, cy = 0;
    std::memset(&in.lens, 0, sizeof(in.lens));
    double* k = in.lens.k; double* p = in.lens.p;
    switch (m->id) {
    case 0: fx = fy = q[0]; cx = q[1]; cy = q[2]; break;                                                     // f cx cy
    case 1: fx = q[0]; fy = q[1]; cx = q[2]; cy = q[3]; break;                                               // fx fy cx cy
    case 2: fx = fy = q[0]; cx = q[1]; cy = q[2]; k[0] = q[3]; break;                                        // f cx cy k
    case 3: fx = fy = q[0]; cx = q[1]; cy = q[2]; k[0] = q[3]; k[1] = q[4]; break;                           // f cx cy k1 k2
    case 4: fx = q[0]; fy = q[1]; cx = q[2]; cy = q[3]; k[0] = q[4]; k[1] = q[5]; p[0] = q[6]; p[1] = q[7]; break;   // .. k1 k2 p1 p2
    case 6: fx = q[0]; fy = q[1]; cx = q[2]; cy = q[3]; k[0] = q[4]; k[1] = q[5]; p[0] = q[6]; p[1] = q[7];          // .. k3 k4 k5 k6
        k[2] = q[8]; k[3] = q[9]; k[4] = q[10]; k[5] = q[11]; break;
    case 5: fx = q[0]; fy = q[1]; cx = q[2]; cy = q[3]; for (int j = 0; j < 4; ++j) k[j] = q[4 + j]; break;  // fx fy cx cy k1..k4
    case 8: fx = fy = q[0]; cx = q[1]; cy = q[2]; k[0] = q[3]; break;                                        // f cx cy k
    case 9: fx = fy = q[0]; cx = q[1]; cy = q[2]; k[0] = q[3]; k[1] = q[4]; break;                           // f cx cy k1 k2
    }
    in.lens.model = m->lens == 2 ? LensDistortion::FISHEYE : LensDistortion::RADTAN;
    in.K = zero3();
    in.K(0, 0) = fx; in.K(0, 2) = cx; in.K(1, 1) = fy; in.K(1, 2) = cy; in.K(2, 2) = 1.0;
    const bool radtan = m->lens == 1;                                   // FULL_OPENCV's k4..k6 only reach the lens (main_colmap.cpp:210)
    in.radial[0] = radtan ? k[0] : 0.0; in.radial[1] = radtan ? k[1] : 0.0; in.radial[2] = radtan ? k[2] : 0.0;
    in.tangential[0] = radtan ? p[0] : 0.0; in.tangential[1] = radtan ? p[1] : 0.0;
    return true;
}

// bounds-checked little-endian reads of one COLMAP binary file, loaded whole (its size bounds every allocation)
struct ColmapBin {
    std::string path;
    std::vector<unsigned char> b;
    size_t pos = 0;
    std::string* error;
    bool bad(const std::string& why) { return fail(error, path + ": " + why); }
    bool open()
    {
        std::ifstream f(path.c_str(), std::ios::binary);
        if (!f) return bad("cannot open");
        b.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
        return true;
    }
    template <class T> bool get(T& v, const char* what)
    {
        if (b.size() - pos < sizeof(T)) return bad(std::string("truncated at byte ") + std::to_string(pos) + " (" + what + ")");
        std::memcpy(&v, b.data() + pos, sizeof(T)); pos += sizeof(T);
        return true;
    }
    bool skip(size_t n, const char* what)
    {
        if (b.size() - pos < n) return bad(std::string("truncated at byte ") + std::to_string(pos) + " (" + what + ")");
        pos += n;
        return true;
    }
    // a record count: each record takes at least min_bytes, so a count the rest of the file cannot hold is malformed
    bool count(uint64_t& n, size_t min_bytes, const char* what)
    {
        if (!get(n, what)) return false;
        if (n > (b.size() - pos) / min_bytes) return bad(std::string(what) + " " + std::to_string(n) + " exceeds what the file holds");
        return true;
    }
    bool name(std::string& s)
    {
        const void* z = std::memchr(b.data() + pos, 0, b.size() - pos);
        if (!z) return bad("unterminated image name at byte " + std::to_string(pos));
        const size_t n = (const unsigned char*)z - (b.data() + pos);
        s.assign((const char*)b.data() + pos, n); pos += n + 1;
        return true;
    }
    bool id32(uint64_t v, unsigned int& out, const char* what)
    {
        if (v > 0xFFFFFFFFull) return bad(std::string(what) + " " + std::to_string(v) + " does not fit unsigned int");
        out = (unsigned int)v;
        return true;
    }
};

static bool file_exists(const std::string& p) { std::ifstream f(p.c_str()); return (bool)f; }

bool readColmap(const std::string& folder, std::vector<SfMCamera>& cams, std::string* error, std::vector<LensDistortion>* lenses)
{
    cams.clear();
    if (lenses) lenses->clear();
    const bool text = file_exists(folder + "/cameras.txt") && file_exists(folder + "/images.txt") && file_exists(folder + "/points3D.txt");
    const bool binary = file_exists(folder + "/cameras.bin") && file_exists(folder + "/images.bin") && file_exists(folder + "/points3D.bin");
    if (!text && !binary) return fail(error, "at least one of the colmap result files does not exist in sfm folder: " + folder);
    std::map<unsigned int, Intrinsics> intr;
    std::map<unsigned int, Vector3d> wps;        // world points referenced by a kept image; (0,0,0) until points3D fills them in
    // one image of images.txt / .bin: kept (and its camera's lens recorded) when its camera is known
    auto add_image = [&](unsigned int img, double qw, double qx, double qy, double qz, double tx, double ty, double tz, unsigned int cam,
                         const std::string& name) {
        std::map<unsigned int, Intrinsics>::const_iterator it = intr.find(cam);
        if (it == intr.end()) return false;
        SfMCamera c = empty_camera(img);
        c.image = name; c.K = it->second.K;
        for (int k = 0; k < 3; ++k) c.radial[k] = it->second.radial[k];
        c.tangential[0] = it->second.tangential[0]; c.tangential[1] = it->second.tangential[1];
        c.R = Line3D::rotationFromQ(qw, qx, qy, qz); c.t = Vector3d(tx, ty, tz); c.C = center_of(c.R, c.t);
        cams.push_back(c);
        if (lenses) lenses->push_back(it->second.lens);
        return true;
    };
    auto add_observation = [&](unsigned int wp) { cams.back().worldpoints.push_back(wp); wps[wp] = Vector3d(0, 0, 0); };
    if (text) {
        std::ifstream fc((folder + "/cameras.txt").c_str()), fi((folder + "/images.txt").c_str()), fp((folder + "/points3D.txt").c_str());
        std::string line;
        while (std::getline(fc, line)) {         // main_colmap.cpp:160-234
            if (line.empty() || line[0] == '#') continue;
            std::stringstream s(line);
            unsigned int cam = 0, w = 0, h = 0; std::string model;
            s >> cam >> model >> w >> h;
            const ColmapModel* m = nullptr;
            for (const ColmapModel& e : kColmapModels) if (model == e.name) m = &e;
            double q[16] = {0};
            for (int k = 0; m && k < m->num_params; ++k) s >> q[k];
            Intrinsics in;
            if (!colmap_intrinsics(m, model, cam, q, lenses != nullptr, in, error)) return false;
            intr[cam] = in;
        }
        bool first = true, keep = false;
        while (std::getline(fi, line)) {         // main_colmap.cpp:252-321: two lines per image
            if (!line.empty() && line[0] == '#') continue;
            std::stringstream s(line);
            if (first) {
                unsigned int img = 0, cam = 0; double qw = 1, qx = 0, qy = 0, qz = 0, tx = 0, ty = 0, tz = 0; std::string name;
                s >> img >> qw >> qx >> qy >> qz >> tx >> ty >> tz >> cam >> name;
                keep = add_image(img, qw, qx, qy, qz, tx, ty, tz, cam, name);
                first = false;
            } else {
                if (keep) {
                    double x, y; std::string id;
                    while (s >> x >> y >> id) {
                        const int wp = std::atoi(id.c_str());
                        if (wp >= 0) add_observation((unsigned int)wp);
                    }
                }
                first = true;
            }
        }
        while (std::getline(fp, line)) {         // main_colmap.cpp:330-349
            if (line.empty() || line[0] == '#') continue;
            std::stringstream s(line);
            unsigned int id = 0; double X = 0, Y = 0, Z = 0;
            s >> id >> X >> Y >> Z;
            std::map<unsigned int, Vector3d>::iterator it = wps.find(id);
            if (s && it != wps.end()) it->second = Vector3d(X, Y, Z);
        }
    } else {                                     // COLMAP's binary model (colmap/scene/reconstruction_io.cc), little-endian
        ColmapBin fc{folder + "/cameras.bin", {}, 0, error}, fi{folder + "/images.bin", {}, 0, error}, fp{folder + "/points3D.bin", {}, 0, error};
        if (!fc.open() || !fi.open() || !fp.open()) return false;
        uint64_t n = 0;
        if (!fc.count(n, 24, "camera count")) return false;
        for (uint64_t i = 0; i < n; ++i) {       // u32 camera_id, i32 model_id, u64 width, u64 height, f64 params[num_params]
            uint32_t cam = 0; int32_t mid = 0; uint64_t w = 0, h = 0;
            if (!fc.get(cam, "camera_id") || !fc.get(mid, "model_id") || !fc.get(w, "width") || !fc.get(h, "height")) return false;
            const ColmapModel* m = nullptr;
            for (const ColmapModel& e : kColmapModels) if (mid == e.id) m = &e;
            if (!m) return fc.bad("camera model id " + std::to_string(mid) + " of camera " + std::to_string(cam) + " unknown!");
            double q[16] = {0};
            for (int k = 0; k < m->num_params; ++k) if (!fc.get(q[k], "camera parameters")) return false;
            Intrinsics in;
            if (!colmap_intrinsics(m, m->name, cam, q, lenses != nullptr, in, error)) return false;
            intr[cam] = in;
        }
        if (!fi.count(n, 4 + 56 + 4 + 1 + 8, "image count")) return false;
        for (uint64_t i = 0; i < n; ++i) {       // u32 image_id, f64 qw qx qy qz tx ty tz, u32 camera_id, name\0, u64 n2d, n2d x (f64 x, f64 y, u64 id)
            uint32_t img = 0, cam = 0; double v[7]; std::string name; uint64_t n2d = 0;
            if (!fi.get(img, "image_id")) return false;
            for (int k = 0; k < 7; ++k) if (!fi.get(v[k], "image pose")) return false;
            if (!fi.get(cam, "camera_id") || !fi.name(name) || !fi.count(n2d, 24, "point count")) return false;
            const bool keep = add_image(img, v[0], v[1], v[2], v[3], v[4], v[5], v[6], cam, name);
            for (uint64_t j = 0; j < n2d; ++j) {
                uint64_t id = 0;
                if (!fi.skip(16, "point xy") || !fi.get(id, "point3D_id")) return false;
                unsigned int wp = 0;
                if (id == ~0ull) continue;       // no 3D point (-1 in images.txt)
                if (!fi.id32(id, wp, "point3D_id")) return false;
                if (keep) add_observation(wp);
            }
        }
        if (!fp.count(n, 8 + 24 + 3 + 8 + 8, "point count")) return false;
        for (uint64_t i = 0; i < n; ++i) {       // u64 id, f64 xyz, u8 rgb, f64 error, u64 track_len, track_len x (u32 image_id, u32 point2D_idx)
            uint64_t id = 0, track = 0; double X = 0, Y = 0, Z = 0;
            unsigned int wp = 0;
            if (!fp.get(id, "point3D_id") || !fp.id32(id, wp, "point3D_id") || !fp.get(X, "xyz") || !fp.get(Y, "xyz") || !fp.get(Z, "xyz") ||
                !fp.skip(3 + 8, "colour and error") || !fp.count(track, 8, "track length") || !fp.skip(8 * (size_t)track, "track"))
                return false;
            std::map<unsigned int, Vector3d>::iterator it = wps.find(wp);
            if (it != wps.end()) it->second = Vector3d(X, Y, Z);
        }
    }
    for (SfMCamera& c : cams) {                  // main_colmap.cpp:386-401
        std::vector<float> d;
        for (unsigned int w : c.worldpoints) d.push_back(point_depth(c.C, wps[w]));
        c.median_depth = median_of(d);
    }
    if (cams.empty()) { if (lenses) lenses->clear(); return fail(error, "no usable image in " + folder); }
    return true;
}

// ------------------------------------------------------------------------------------------------ mavmap
bool readMavmap(const std::string& path, std::vector<SfMCamera>& out, std::string* error)
{
    out.clear();
    std::vector<SfMCamera> cams;                  // handed out only when the whole file has been read
    std::ifstream f(path.c_str());
    if (!f) return fail(error, "cannot open " + path);
    std::string line;
    long long lineno = 0;
    bool have = false;
    while (std::getline(f, line)) {               // main_mavmap.cpp:158-162: leading comment lines
        ++lineno;
        if (line.substr(0, 1) != "#") { have = true; break; }
    }
    for (; have; have = (bool)std::getline(f, line), ++lineno) {
        if (line.length() < 28) break;            // main_mavmap.cpp:172-173
        const std::string where = path + ":" + std::to_string(lineno) + ": ";
        std::istringstream s(line);
        std::string tok[17];                      // filename roll pitch yaw lat lon alt h tx ty tz camID camModel fx fy cx cy
        for (int k = 0; k < 17; ++k)
            if (!(s >> tok[k])) return fail(error, where + "truncated camera line (" + std::to_string(k) + " of 17 fields)");
        auto strip = [](const std::string& x) { return x.substr(0, x.length() - 1); };     // every field ends with a comma
        if (strip(tok[12]) != "PINHOLE") return fail(error, where + "camera model '" + strip(tok[12]) + "': only PINHOLE camera model supported");
        static const int num_idx[10] = {1, 2, 3, 8, 9, 10, 13, 14, 15, 16};
        double v[17];
        for (int k : num_idx)
            if (!to_double(strip(tok[k]), v[k])) return fail(error, where + "non-numeric field " + std::to_string(k + 1) + " '" + tok[k] + "'");
        SfMCamera c = empty_camera((unsigned int)cams.size());
        c.image = strip(tok[0]);
        const Matrix3d R = Line3D::rotationFromRPY(v[1], v[2], v[3]);
        for (int r = 0; r < 3; ++r)               // [R|t]^-1 = [R^T | -R^T t]  (main_mavmap.cpp:214-223)
            for (int k = 0; k < 3; ++k) c.R(r, k) = R(k, r);
        c.C = Vector3d(v[8], v[9], v[10]);        // mavmap stores the camera centre
        c.t = translation_of(c.R, c.C);
        c.K(0, 0) = v[13]; c.K(1, 1) = v[14]; c.K(0, 2) = v[15]; c.K(1, 2) = v[16]; c.K(2, 2) = 1.0;     // main_mavmap.cpp:290-296
        cams.push_back(c);
    }
    if (cams.empty()) return fail(error, "no camera in mavmap file " + path);
    out.swap(cams);
    return true;
}

// ------------------------------------------------------------------------------------------------ JSON (OpenMVG's sfm_data.json)
// A validating cursor over the document text: the whole document is checked once (syntax, nesting depth), then values are found by
// scanning objects and arrays in place.  Nothing is copied but the strings that are read and no tree is built, so memory stays at
// the size of the file.
static const int JSON_MAX_DEPTH = 64;

struct Json {
    const char* b = nullptr;
    const char* e = nullptr;
    std::string err;
    static const char* ws(const char* p, const char* e) { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) ++p; return p; }
    long long line_of(const char* p) const { return 1 + std::count(b, p, '\n'); }
    bool bad(const char* p, const char* what) { err = "line " + std::to_string(line_of(p)) + ": " + what; return false; }

    // string starting at p ('"'); out (optional) gets the decoded UTF-8; p is left after the closing quote
    bool str(const char*& p, std::string* out)
    {
        const char* s = p++;
        while (true) {
            if (p >= e) return bad(s, "unterminated string");
            const unsigned char ch = (unsigned char)*p;
            if (ch == '"') { ++p; return true; }
            if (ch < 0x20) return bad(p, "control character in a string");
            if (ch != '\\') { if (out) out->push_back((char)ch); ++p; continue; }
            if (++p >= e) return bad(s, "unterminated string");
            const char x = *p++;
            switch (x) {
            case '"': case '\\': case '/': if (out) out->push_back(x); break;
            case 'b': if (out) out->push_back('\b'); break;
            case 'f': if (out) out->push_back('\f'); break;
            case 'n': if (out) out->push_back('\n'); break;
            case 'r': if (out) out->push_back('\r'); break;
            case 't': if (out) out->push_back('\t'); break;
            case 'u': {
                unsigned cp = 0;
                if (!hex4(p, cp)) return bad(p, "bad \\u escape");
                if (cp >= 0xD800 && cp < 0xDC00) {          // surrogate pair
                    unsigned lo = 0;
                    if (e - p < 2 || p[0] != '\\' || p[1] != 'u') return bad(p, "unpaired surrogate");
                    p += 2;
                    if (!hex4(p, lo) || lo < 0xDC00 || lo >= 0xE000) return bad(p, "unpaired surrogate");
                    cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                } else if (cp >= 0xDC00 && cp < 0xE000) return bad(p, "unpaired surrogate");
                if (out) utf8(cp, *out);
                break;
            }
            default: return bad(p - 1, "bad escape in a string");
            }
        }
    }
    bool hex4(const char*& p, unsigned& v)
    {
        if (e - p < 4) return false;
        v = 0;
        for (int i = 0; i < 4; ++i, ++p) {
            const char c = *p;
            v <<= 4;
            if (c >= '0' && c <= '9') v |= (unsigned)(c - '0');
            else if (c >= 'a' && c <= 'f') v |= (unsigned)(c - 'a' + 10);
            else if (c >= 'A' && c <= 'F') v |= (unsigned)(c - 'A' + 10);
            else return false;
        }
        return true;
    }
    static void utf8(unsigned cp, std::string& o)
    {
        if (cp < 0x80) o.push_back((char)cp);
        else if (cp < 0x800) { o.push_back((char)(0xC0 | (cp >> 6))); o.push_back((char)(0x80 | (cp & 63))); }
        else if (cp < 0x10000) { o.push_back((char)(0xE0 | (cp >> 12))); o.push_back((char)(0x80 | ((cp >> 6) & 63))); o.push_back((char)(0x80 | (cp & 63))); }
        else { o.push_back((char)(0xF0 | (cp >> 18))); o.push_back((char)(0x80 | ((cp >> 12) & 63))); o.push_back((char)(0x80 | ((cp >> 6) & 63))); o.push_back((char)(0x80 | (cp & 63))); }
    }
    // a number token (RFC 8259 grammar) starting at p; p is left after it
    bool num(const char*& p)
    {
        const char* s = p;
        if (p < e && *p == '-') ++p;
        if (p < e && *p == '0') ++p;
        else if (p < e && *p >= '1' && *p <= '9') while (p < e && *p >= '0' && *p <= '9') ++p;
        else return bad(s, "bad number");
        if (p < e && *p == '.') { ++p; if (p >= e || *p < '0' || *p > '9') return bad(s, "bad number"); while (p < e && *p >= '0' && *p <= '9') ++p; }
        if (p < e && (*p == 'e' || *p == 'E')) {
            ++p;
            if (p < e && (*p == '+' || *p == '-')) ++p;
            if (p >= e || *p < '0' || *p > '9') return bad(s, "bad number");
            while (p < e && *p >= '0' && *p <= '9') ++p;
        }
        return true;
    }
    // skips (and checks) the value at p; p is left after it
    bool skip(const char*& p, int depth)
    {
        p = ws(p, e);
        if (p >= e) return bad(p, "unexpected end of the document");
        const char c = *p;
        if (c == '"') return str(p, nullptr);
        if (c == '{' || c == '[') {
            if (depth >= JSON_MAX_DEPTH) return bad(p, "nesting deeper than 64 levels");
            const char close = c == '{' ? '}' : ']';
            p = ws(p + 1, e);
            if (p < e && *p == close) { ++p; return true; }
            while (true) {
                if (c == '{') {
                    p = ws(p, e);
                    if (p >= e || *p != '"') return bad(p, "expected a member name");
                    if (!str(p, nullptr)) return false;
                    p = ws(p, e);
                    if (p >= e || *p != ':') return bad(p, "expected ':'");
                    ++p;
                }
                if (!skip(p, depth + 1)) return false;
                p = ws(p, e);
                if (p < e && *p == ',') { ++p; continue; }
                if (p < e && *p == close) { ++p; return true; }
                return bad(p, c == '{' ? "expected ',' or '}'" : "expected ',' or ']'");
            }
        }
        if (c == '-' || (c >= '0' && c <= '9')) return num(p);
        for (const char* lit : {"true", "false", "null"}) {
            const size_t n = std::strlen(lit);
            if ((size_t)(e - p) >= n && std::memcmp(p, lit, n) == 0) { p += n; return true; }
        }
        return bad(p, "unexpected character");
    }
    // the following assume a checked document
    static const char* after(const char* p, const char* e) { Json j; j.b = p; j.e = e; j.skip(p, 0); return p; }
};

// a value inside a checked document: its position and its JSON path (for messages)
struct JV {
    const Json* J = nullptr;
    const char* p = nullptr;     // first character of the value; nullptr: the member does not exist
    std::string path;
    char type() const { return p ? *p : 0; }
    bool is_obj() const { return type() == '{'; }
    bool is_arr() const { return type() == '['; }
    bool is_str() const { return type() == '"'; }
    bool is_num() const { return type() == '-' || (type() >= '0' && type() <= '9'); }
    // member `key` of an object (the first one if the name repeats, as rapidjson's operator[] finds it)
    JV operator[](const char* key) const
    {
        JV r{J, nullptr, path + "." + key};
        if (!is_obj()) return r;
        const char* q = Json::ws(p + 1, J->e);
        while (q < J->e && *q == '"') {
            std::string name;
            Json tmp; tmp.b = J->b; tmp.e = J->e;
            tmp.str(q, &name);
            q = Json::ws(q, J->e) + 1;                 // ':'
            q = Json::ws(q, J->e);
            if (name == key) { r.p = q; return r; }
            q = Json::ws(Json::after(q, J->e), J->e);
            if (*q == ',') q = Json::ws(q + 1, J->e);
        }
        return r;
    }
    // the elements of an array
    std::vector<JV> elements() const
    {
        std::vector<JV> v;
        if (!is_arr()) return v;
        const char* q = Json::ws(p + 1, J->e);
        if (*q == ']') return v;
        for (size_t i = 0;; ++i) {
            v.push_back(JV{J, q, path + "[" + std::to_string(i) + "]"});
            q = Json::ws(Json::after(q, J->e), J->e);
            if (*q != ',') break;
            q = Json::ws(q + 1, J->e);
        }
        return v;
    }
};

struct JsonReader {
    std::string file;
    std::string* error;
    bool ok = true;
    bool fail_at(const JV& v, const std::string& what)
    {
        if (ok) fail(error, file + ": " + v.path + ": " + (v.p ? what : "missing"));
        ok = false;
        return false;
    }
    bool need(const JV& v, bool (JV::*is)() const, const char* what) { return v.p && (v.*is)() ? true : fail_at(v, std::string("expected ") + what); }
    bool dbl(const JV& v, double& out)
    {
        if (!need(v, &JV::is_num, "a number")) return false;
        out = std::strtod(v.p, nullptr);      // the token is a checked JSON number, followed by a non-number character
        return true;
    }
    // rapidjson's GetUint: an integer token (no fraction, no exponent) in [0, 2^32)
    bool uint(const JV& v, unsigned int& out)
    {
        if (!need(v, &JV::is_num, "an unsigned integer")) return false;
        const char* q = v.p;
        unsigned long long x = 0;
        while (*q >= '0' && *q <= '9') { x = x * 10 + (unsigned)(*q - '0'); if (x > 0xFFFFFFFFull) return fail_at(v, "unsigned integer out of range"); ++q; }
        if (q == v.p || *q == '.' || *q == 'e' || *q == 'E') return fail_at(v, "expected an unsigned integer");
        out = (unsigned int)x;
        return true;
    }
    bool string(const JV& v, std::string& out)
    {
        if (!need(v, &JV::is_str, "a string")) return false;
        const char* q = v.p;
        Json tmp; tmp.b = v.J->b; tmp.e = v.J->e;
        out.clear();
        return tmp.str(q, &out);
    }
    bool array(const JV& v, std::vector<JV>& out) { if (!need(v, &JV::is_arr, "an array")) return false; out = v.elements(); return true; }
    // element i of an array value
    bool at(const JV& v, size_t i, JV& out)
    {
        std::vector<JV> el;
        if (!array(v, el)) return false;
        if (i >= el.size()) return fail_at(JV{v.J, v.p, v.path + "[" + std::to_string(i) + "]"}, "missing");
        out = el[i];
        return true;
    }
    bool dbl_at(const JV& v, size_t i, double& out) { JV x; return at(v, i, x) && dbl(x, out); }
};

bool readOpenMVG(const std::string& path, std::vector<SfMCamera>& cams, std::string* error)
{
    cams.clear();
    std::ifstream f(path.c_str(), std::ios::binary);
    if (!f) return fail(error, "cannot open " + path);
    std::string text((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    Json J;
    J.b = text.c_str(); J.e = J.b + text.size();
    const char* p = J.b;
    if (!J.skip(p, 0)) return fail(error, path + ": " + J.err);
    if (Json::ws(p, J.e) != J.e) return fail(error, path + ": line " + std::to_string(J.line_of(p)) + ": text after the JSON document");
    JsonReader rd{path, error};
    const JV root{&J, Json::ws(J.b, J.e), ""};
    if (!rd.need(root, &JV::is_obj, "an object")) return false;

    // views (main_openmvg.cpp:152-199).  The reader does not look for the images: a frontend skips a view whose image it cannot load.
    struct View { unsigned int id, intr, pose; std::string file; };
    std::vector<View> views;
    std::map<unsigned int, unsigned int> pose2view;
    std::vector<JV> arr;
    if (!rd.array(root["views"], arr)) return false;
    if (arr.empty()) return fail(error, path + ": No aligned cameras in json file!");
    for (const JV& el : arr) {
        const JV d = el["value"]["ptr_wrapper"]["data"];
        View v;
        if (!rd.string(d["filename"], v.file) || !rd.uint(d["id_view"], v.id) || !rd.uint(d["id_intrinsic"], v.intr) || !rd.uint(d["id_pose"], v.pose)) return false;
        views.push_back(v);
        pose2view[v.pose] = v.id;
    }

    // intrinsics (main_openmvg.cpp:201-277).  cam_model lives outside the loop in the reference: an entry without polymorphic_name
    // keeps the model of the entry before it (none before the first: no distortion)
    std::map<unsigned int, Intrinsics> intr;
    if (!rd.array(root["intrinsics"], arr)) return false;
    if (arr.empty()) return fail(error, path + ": No intrinsics in json file!");
    std::string model;
    for (const JV& el : arr) {
        const JV val = el["value"], d = val["ptr_wrapper"]["data"];
        if (val["polymorphic_name"].p && !rd.string(val["polymorphic_name"], model)) return false;
        unsigned int key = 0;
        double focal = 0, px = 0, py = 0;
        Intrinsics in;
        std::memset(&in, 0, sizeof(in));
        if (!rd.uint(el["key"], key) || !rd.dbl(d["focal_length"], focal) || !rd.dbl_at(d["principal_point"], 0, px) || !rd.dbl_at(d["principal_point"], 1, py))
            return false;
        if (model == "pinhole_radial_k3") { for (int k = 0; k < 3; ++k) if (!rd.dbl_at(d["disto_k3"], k, in.radial[k])) return false; }
        else if (model == "pinhole_radial_k1") { if (!rd.dbl_at(d["disto_k1"], 0, in.radial[0])) return false; }
        else if (model == "pinhole_brown_t2") {
            for (int k = 0; k < 3; ++k) if (!rd.dbl_at(d["disto_t2"], k, in.radial[k])) return false;
            for (int k = 0; k < 2; ++k) if (!rd.dbl_at(d["disto_t2"], 3 + k, in.tangential[k])) return false;
        }                                         // any other model: no distortion (the reference warns unless it is "pinhole")
        in.K(0, 0) = focal; in.K(1, 1) = focal; in.K(0, 2) = px; in.K(1, 2) = py; in.K(2, 2) = 1.0;
        intr[key] = in;
    }

    // extrinsics (main_openmvg.cpp:279-324): t = -R C
    struct Pose { Matrix3d R; Vector3d t, C; };
    std::map<unsigned int, Pose> poses;           // by view id
    if (!rd.array(root["extrinsics"], arr)) return false;
    if (arr.empty()) return fail(error, path + ": No extrinsics in json file!");
    for (const JV& el : arr) {
        unsigned int key = 0;
        if (!rd.uint(el["key"], key)) return false;
        std::map<unsigned int, unsigned int>::const_iterator it = pose2view.find(key);
        if (it == pose2view.end()) continue;      // a pose no view uses
        const JV val = el["value"];
        Pose ps;
        for (int r = 0; r < 3; ++r) {
            JV row;
            if (!rd.at(val["rotation"], r, row)) return false;
            for (int c = 0; c < 3; ++c) if (!rd.dbl_at(row, c, ps.R(r, c))) return false;
        }
        if (!rd.dbl_at(val["center"], 0, ps.C.x) || !rd.dbl_at(val["center"], 1, ps.C.y) || !rd.dbl_at(val["center"], 2, ps.C.z)) return false;
        ps.t = translation_of(ps.R, ps.C);
        poses[it->second] = ps;
    }

    // structure (main_openmvg.cpp:326-365): per view the world point ids and float depths |C - X| in file order
    std::map<unsigned int, std::list<unsigned int> > wps;
    std::map<unsigned int, std::vector<float> > depths;
    if (!rd.array(root["structure"], arr)) return false;
    if (arr.empty()) return fail(error, path + ": No worldpoints in json file!");
    std::vector<JV> obs;
    for (const JV& el : arr) {
        unsigned int id = 0;
        Vector3d X;
        const JV val = el["value"];
        if (!rd.uint(el["key"], id)) return false;
        if (!rd.dbl_at(val["X"], 0, X.x) || !rd.dbl_at(val["X"], 1, X.y) || !rd.dbl_at(val["X"], 2, X.z)) return false;
        if (!rd.array(val["observations"], obs)) return false;
        for (const JV& o : obs) {
            unsigned int view = 0;
            if (!rd.uint(o["key"], view)) return false;
            std::map<unsigned int, Pose>::const_iterator it = poses.find(view);
            if (it == poses.end()) continue;
            wps[view].push_back(id);
            depths[view].push_back(point_depth(it->second.C, X));
        }
    }

    // cameras in view order (main_openmvg.cpp:367-409)
    for (const View& v : views) {
        if (!wps.count(v.id) || !intr.count(v.intr)) continue;
        const Intrinsics& in = intr[v.intr];
        const Pose& ps = poses[v.id];
        SfMCamera c = empty_camera(v.id);
        c.image = v.file; c.K = in.K;
        for (int k = 0; k < 3; ++k) c.radial[k] = in.radial[k];
        c.tangential[0] = in.tangential[0]; c.tangential[1] = in.tangential[1];
        c.R = ps.R; c.t = ps.t; c.C = ps.C;
        c.worldpoints = wps[v.id];
        c.median_depth = median_of(depths[v.id]);
        cams.push_back(c);
    }
    if (cams.empty()) return fail(error, path + ": no view has both intrinsics and world points");
    return true;
}

// ------------------------------------------------------------------------------------------------ Pix4D
bool readPix4D(const std::string& params_folder, const std::string& project_prefix, std::vector<SfMCamera>& out, std::string* error, int cuda_device)
{
    out.clear();
    std::vector<SfMCamera> cams;                  // handed out only when everything has been read
    std::string prefix = params_folder + "/" + project_prefix;          // main_pix4d.cpp:163-166
    if (prefix.substr(prefix.length() - 1, 1) != "_") prefix += "_";
    const std::string file1 = prefix + "calibrated_camera_parameters.txt", file2 = prefix + "tp_pix4d.txt";
    std::ifstream fc(file1.c_str()), fp(file2.c_str());
    if (!fc || !fp) return fail(error, "pix4d file '" + file1 + "' or '" + file2 + "' does not exist!");

    // calibrated_camera_parameters.txt (main_pix4d.cpp:185-276)
    std::string line;
    long long lineno = 0;
    while (std::getline(fc, line)) { ++lineno; if (line.length() < 2) break; }    // the description block
    std::map<std::string, size_t> img2pos;
    std::vector<std::string> rawnames;
    std::vector<double> P;                        // 12 per camera, K [R|t] row-major
    while (std::getline(fc, line)) {
        ++lineno;
        if (line.length() < 5) break;
        const long long head = lineno;
        std::istringstream s(line);
        std::string fname;
        s >> fname;
        SfMCamera c = empty_camera((unsigned int)cams.size());
        c.image = fname;
        double v[3];
        auto next = [&](int n, const char* what) -> bool {
            if (!std::getline(fc, line)) return fail(error, file1 + ":" + std::to_string(head) + ": camera block of '" + fname + "' is truncated (no " + what + ")");
            ++lineno;
            if (!read_numbers(line, v, n)) return fail(error, file1 + ":" + std::to_string(lineno) + ": expected " + std::to_string(n) + " numbers (" + what + ")");
            return true;
        };
        for (int r = 0; r < 3; ++r) { if (!next(3, "K row")) return false; for (int k = 0; k < 3; ++k) c.K(r, k) = v[k]; }
        if (!next(3, "radial distortion")) return false;
        for (int k = 0; k < 3; ++k) c.radial[k] = v[k];
        if (!next(2, "tangential distortion")) return false;
        c.tangential[0] = v[0]; c.tangential[1] = v[1];
        if (!next(3, "camera centre")) return false;
        const Vector3d centre(v[0], v[1], v[2]);
        for (int r = 0; r < 3; ++r) { if (!next(3, "R row")) return false; for (int k = 0; k < 3; ++k) c.R(r, k) = v[k]; }
        const Matrix3d& R = c.R;
        c.t = translation_of(R, centre);
        c.C = mul_transposed(R, neg(c.t));        // R^T (-t) as main_pix4d.cpp:391-392 forms it, not center_of's -(R^T t)
        const double Rt[12] = {R(0, 0), R(0, 1), R(0, 2), c.t.x, R(1, 0), R(1, 1), R(1, 2), c.t.y, R(2, 0), R(2, 1), R(2, 2), c.t.z};
        for (int r = 0; r < 3; ++r)
            for (int k = 0; k < 4; ++k) P.push_back(c.K(r, 0) * Rt[k] + c.K(r, 1) * Rt[4 + k] + c.K(r, 2) * Rt[8 + k]);
        const size_t dot = fname.find_last_of(".");
        rawnames.push_back(fname.substr(0, dot));
        img2pos[rawnames.back()] = cams.size();
        cams.push_back(c);
    }
    if (cams.empty()) return fail(error, file1 + ": no camera");

    // tp_pix4d.txt (main_pix4d.cpp:282-349): key-image lines and "id x y scale" observation lines; ids starting with '-' are skipped
    std::map<std::string, unsigned int> feat_id;
    std::map<std::string, std::list<unsigned int> > per_key;
    std::vector<long long> obs_count;             // per feature, then the CSR offsets
    std::vector<std::pair<unsigned int, unsigned int> > obs_feat_cam;
    std::vector<double> obs_xy;
    std::string key;
    bool have_key = false;
    size_t key_pos = 0;
    lineno = 0;
    while (std::getline(fp, line)) {
        ++lineno;
        std::istringstream s(line);
        std::string id, rest;
        s >> id >> rest;
        if (id.length() < 2) break;
        if (id[0] == '-') continue;
        if (rest.empty()) {
            key = id; have_key = true;
            key_pos = img2pos[key];                // a name missing from the camera file becomes camera 0 (std::map::operator[])
            continue;
        }
        if (!have_key) return fail(error, file2 + ":" + std::to_string(lineno) + ": observation before the first key image");
        double xy[2];
        std::istringstream s2(line);
        std::string t0, tx, ty;
        s2 >> t0 >> tx >> ty;
        if (!to_double(tx, xy[0]) || !to_double(ty, xy[1])) return fail(error, file2 + ":" + std::to_string(lineno) + ": non-numeric image coordinates");
        std::map<std::string, unsigned int>::iterator it = feat_id.find(id);
        unsigned int fid;
        if (it == feat_id.end()) { fid = (unsigned int)obs_count.size(); feat_id[id] = fid; obs_count.push_back(0); }
        else fid = it->second;
        per_key[key].push_back(fid);
        ++obs_count[fid];
        obs_feat_cam.push_back(std::make_pair(fid, (unsigned int)key_pos));
        obs_xy.push_back(xy[0]); obs_xy.push_back(xy[1]);
    }
    // observations grouped by feature, in file order within each feature
    const size_t n_pts = obs_count.size(), n_obs = obs_feat_cam.size();
    std::vector<int64_t> ptr(n_pts + 1, 0);
    for (size_t i = 0; i < n_pts; ++i) ptr[i + 1] = ptr[i] + obs_count[i];
    std::vector<int64_t> fill(ptr.begin(), ptr.end() - 1);
    std::vector<int32_t> ocam(n_obs);
    std::vector<double> oxy(2 * n_obs);
    for (size_t o = 0; o < n_obs; ++o) {
        const int64_t k = fill[obs_feat_cam[o].first]++;
        ocam[k] = (int32_t)obs_feat_cam[o].second;
        oxy[2 * k] = obs_xy[2 * o]; oxy[2 * k + 1] = obs_xy[2 * o + 1];
    }
    // per camera: the observations of its key image (duplicates included) and the camera centre
    std::vector<int64_t> lptr(cams.size() + 1, 0);
    std::vector<int32_t> lpts;
    std::vector<double> Cs;
    for (size_t i = 0; i < cams.size(); ++i) {
        std::map<std::string, std::list<unsigned int> >::const_iterator it = per_key.find(rawnames[i]);
        if (it != per_key.end()) {
            cams[i].worldpoints = it->second;
            for (unsigned int w : it->second) lpts.push_back((int32_t)w);
        }
        lptr[i + 1] = (int64_t)lpts.size();
        Cs.push_back(cams[i].C.x); Cs.push_back(cams[i].C.y); Cs.push_back(cams[i].C.z);
    }

    // triangulation and median depths on the GPU (main_pix4d.cpp:354-418)
    l3d_ctx* ctx = nullptr;
    if (l3d_ctx_create(cuda_device, &ctx) != L3D_OK) return fail(error, "readPix4D: no usable CUDA device (the tie points are triangulated on the GPU)");
    std::vector<double> X(3 * n_pts);
    std::vector<int32_t> valid(n_pts), cnt(cams.size());
    std::vector<float> med(cams.size());
    int rc = l3d_triangulate_points(ctx, (long long)n_pts, ptr.data(), ocam.data(), oxy.data(), (int)cams.size(), P.data(), X.data(), valid.data(), 0);
    if (rc == L3D_OK)
        rc = l3d_median_depths(ctx, (int)cams.size(), lptr.data(), lpts.data(), (long long)n_pts, X.data(), valid.data(), Cs.data(), cnt.data(), med.data(), 0);
    const std::string msg = rc == L3D_OK ? "" : std::string("readPix4D: ") + l3d_last_error(ctx);
    l3d_ctx_destroy(ctx);
    if (rc != L3D_OK) return fail(error, msg);
    for (size_t i = 0; i < cams.size(); ++i)      // a camera needs more than two valid points (main_pix4d.cpp:405)
        if (cnt[i] > 2) { cams[i].median_depth = med[i]; out.push_back(cams[i]); }
    if (out.empty()) return fail(error, file2 + ": no camera sees more than two triangulated points");
    return true;
}

// ------------------------------------------------------------------------------------------------ what the C wrappers share
// element i of a handle's list; nullptr when i is out of range
template <class T> static const T* item(const std::vector<T>& v, int i) { return i >= 0 && i < (int)v.size() ? &v[i] : nullptr; }

// a list of ids (world points, neighbours) into out[cap]: its length, even when it exceeds cap
static int copy_ids(const std::list<unsigned int>& ids, unsigned int* out, int cap)
{
    int n = 0;
    for (unsigned int w : ids) { if (n < cap) out[n] = w; ++n; }
    return n;
}

}  // namespace L3DPP

// the object behind an l3dpp_sfm_* handle: the cameras of any reader, and the lenses readColmap returns when asked for them
struct L3DSfMHandle {
    std::vector<L3DPP::SfMCamera> cams;
    std::vector<L3DPP::LensDistortion> lenses;
};
typedef std::vector<L3DPP::NVMCamera> L3DNVMHandle;

// C wrapper (include/l3dpp_capi.h): flat arrays
extern "C" {
void* l3dpp_nvm_open(const char* path, char* err, int errcap)
{
    L3DNVMHandle* v = new L3DNVMHandle();
    std::string e;
    if (!L3DPP::readNVM(path, *v, &e)) { l3dpp_copy_str(e, err, errcap); delete v; return nullptr; }
    return v;
}
void l3dpp_nvm_close(void* h) { delete (L3DNVMHandle*)h; }
int l3dpp_nvm_num_cameras(void* h) { return (int)((L3DNVMHandle*)h)->size(); }
int l3dpp_nvm_camera(void* h, int i, double* R9, double* t3, double* C3, float* focal, float* distortion, float* median_depth, int* num_wps, char* name, int namecap)
{
    const L3DPP::NVMCamera* c = L3DPP::item(*(L3DNVMHandle*)h, i);
    if (!c) return -1;
    for (int k = 0; k < 9; ++k) R9[k] = c->R.m[k];
    t3[0] = c->t.x; t3[1] = c->t.y; t3[2] = c->t.z; C3[0] = c->C.x; C3[1] = c->C.y; C3[2] = c->C.z;
    *focal = c->focal; *distortion = c->distortion; *median_depth = c->median_depth; *num_wps = (int)c->worldpoints.size();
    l3dpp_copy_str(c->image, name, namecap);
    return 0;
}
int l3dpp_nvm_worldpoints(void* h, int i, unsigned int* out, int cap) { const L3DPP::NVMCamera* c = L3DPP::item(*(L3DNVMHandle*)h, i); return c ? L3DPP::copy_ids(c->worldpoints, out, cap) : -1; }
void l3dpp_intrinsics_from_focal(float focal, int w, int h, double* K9) { const L3DPP::Matrix3d K = L3DPP::intrinsicsFromFocal(focal, w, h); for (int k = 0; k < 9; ++k) K9[k] = K.m[k]; }
void* l3dpp_sfm_open(int kind, const char* path, const char* aux, char* err, int errcap)
{
    L3DSfMHandle* v = new L3DSfMHandle();
    const std::string a = aux ? aux : "";
    std::string e;
    bool ok = false;
    switch (kind) {
    case L3DPP_SFM_BUNDLER: ok = L3DPP::readBundler(path, a, v->cams, &e); break;
    case L3DPP_SFM_COLMAP: ok = L3DPP::readColmap(path, v->cams, &e); break;
    case L3DPP_SFM_COLMAP_LENSES: ok = L3DPP::readColmap(path, v->cams, &e, &v->lenses); break;
    case L3DPP_SFM_MAVMAP: ok = L3DPP::readMavmap(path, v->cams, &e); break;
    case L3DPP_SFM_OPENMVG: ok = L3DPP::readOpenMVG(path, v->cams, &e); break;
    case L3DPP_SFM_PIX4D: ok = L3DPP::readPix4D(path, a, v->cams, &e); break;
    default: e = "unknown model kind " + std::to_string(kind);
    }
    if (!ok) { l3dpp_copy_str(e, err, errcap); delete v; return nullptr; }
    return v;
}
void l3dpp_sfm_close(void* h) { delete (L3DSfMHandle*)h; }
int l3dpp_sfm_num_cameras(void* h) { return (int)((L3DSfMHandle*)h)->cams.size(); }
int l3dpp_sfm_lens(void* h, int i, double* lens9)
{
    const L3DPP::LensDistortion* l = L3DPP::item(((L3DSfMHandle*)h)->lenses, i);
    if (!l) return -1;
    lens9[0] = l->model;
    for (int k = 0; k < 6; ++k) lens9[1 + k] = l->k[k];
    lens9[7] = l->p[0]; lens9[8] = l->p[1];
    return 0;
}
int l3dpp_sfm_camera(void* h, int i, double* head5, double* K9, double* R9, double* t3, double* C3, double* dist5, char* name, int namecap)
{
    const L3DPP::SfMCamera* c = L3DPP::item(((L3DSfMHandle*)h)->cams, i);
    if (!c) return -1;
    head5[0] = c->id; head5[1] = c->has_K; head5[2] = c->focal; head5[3] = c->median_depth; head5[4] = (double)c->worldpoints.size();
    for (int k = 0; k < 9; ++k) { K9[k] = c->K.m[k]; R9[k] = c->R.m[k]; }
    t3[0] = c->t.x; t3[1] = c->t.y; t3[2] = c->t.z; C3[0] = c->C.x; C3[1] = c->C.y; C3[2] = c->C.z;
    for (int k = 0; k < 3; ++k) dist5[k] = c->radial[k];
    dist5[3] = c->tangential[0]; dist5[4] = c->tangential[1];
    l3dpp_copy_str(c->image, name, namecap);
    return 0;
}
int l3dpp_sfm_worldpoints(void* h, int i, unsigned int* out, int cap) { const L3DPP::SfMCamera* c = L3DPP::item(((L3DSfMHandle*)h)->cams, i); return c ? L3DPP::copy_ids(c->worldpoints, out, cap) : -1; }
void l3dpp_rotation_from_rpy(double roll, double pitch, double yaw, double* R9)
{
    const L3DPP::Matrix3d R = L3DPP::Line3D::rotationFromRPY(roll, pitch, yaw);
    for (int k = 0; k < 9; ++k) R9[k] = R.m[k];
}
void l3dpp_decompose_projection(const double* P12, double* K9, double* R9, double* t3)
{
    L3DPP::Matrix3d K, R; L3DPP::Vector3d t;
    L3DPP::Line3D::decomposeProjectionMatrix(P12, K, R, t);
    for (int k = 0; k < 9; ++k) { K9[k] = K.m[k]; R9[k] = R.m[k]; }
    t3[0] = t.x; t3[1] = t.y; t3[2] = t.z;
}
int l3dpp_sequential_neighbors(unsigned int i, unsigned int n_cams, unsigned int num_neighbors, unsigned int* out, int cap)
{
    return L3DPP::copy_ids(L3DPP::sequentialNeighbors(i, n_cams, num_neighbors), out, cap);
}
}
