// line3d_io.cc — .nvm, Bundler and COLMAP (text and binary) readers for frontends built on include/line3d.h (restates main_vsfm.cpp:143-310,
// main_bundler.cpp, main_colmap.cpp; host only)
#include "../../include/line3d_io.h"
#include "../../include/l3dpp_capi.h"
#include "l3dpp_wrap.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <cstdint>
#include <fstream>
#include <iterator>
#include <map>
#include <sstream>

namespace L3DPP {

bool readNVM(const std::string& path, std::vector<NVMCamera>& cams, std::string* error)
{
    cams.clear();
    std::ifstream f(path.c_str());
    if (!f) { if (error) *error = "cannot open " + path; return false; }
    std::string line;
    std::getline(f, line);                       // "NVM_V3"
    std::getline(f, line);                       // empty
    std::getline(f, line);
    unsigned int num_cams = 0;
    { std::stringstream s(line); s >> num_cams; }
    if (num_cams == 0) { if (error) *error = "No aligned cameras in NVM file!"; return false; }     // main_vsfm.cpp:157-161
    cams.resize(num_cams);
    for (unsigned int i = 0; i < num_cams; ++i) {
        double focal = 0, qw = 1, qx = 0, qy = 0, qz = 0, Cx = 0, Cy = 0, Cz = 0, dist = 0;
        NVMCamera& c = cams[i];
        // a truncated or malformed camera line must not become a default camera (the reference has the same hole, main_vsfm.cpp:168-190)
        if (!std::getline(f, line)) { if (error) *error = "unexpected end of file in the camera list of " + path + " (camera " + std::to_string(i) + ")"; return false; }
        std::stringstream s(line);
        if (!(s >> c.image >> focal >> qw >> qx >> qy >> qz >> Cx >> Cy >> Cz >> dist)) {
            if (error) *error = "malformed camera line " + std::to_string(i) + " in " + path;
            return false;
        }
        c.focal = (float)focal; c.distortion = (float)dist;
        Matrix3d& R = c.R;                        // main_vsfm.cpp:193-203 (the quaternion is used as stored, not re-normalised)
        R(0, 0) = 1.0 - 2.0 * qy * qy - 2.0 * qz * qz; R(0, 1) = 2.0 * qx * qy - 2.0 * qz * qw; R(0, 2) = 2.0 * qx * qz + 2.0 * qy * qw;
        R(1, 0) = 2.0 * qx * qy + 2.0 * qz * qw; R(1, 1) = 1.0 - 2.0 * qx * qx - 2.0 * qz * qz; R(1, 2) = 2.0 * qy * qz - 2.0 * qx * qw;
        R(2, 0) = 2.0 * qx * qz - 2.0 * qy * qw; R(2, 1) = 2.0 * qy * qz + 2.0 * qx * qw; R(2, 2) = 1.0 - 2.0 * qx * qx - 2.0 * qy * qy;
        c.C = Vector3d(Cx, Cy, Cz);
        c.t = Vector3d(-(R(0, 0) * Cx + R(0, 1) * Cy + R(0, 2) * Cz), -(R(1, 0) * Cx + R(1, 1) * Cy + R(1, 2) * Cz),
                       -(R(2, 0) * Cx + R(2, 1) * Cy + R(2, 2) * Cz));
        c.median_depth = 0.0f;
    }
    std::getline(f, line);                       // empty
    std::getline(f, line);
    unsigned int num_points = 0;
    { std::stringstream s(line); s >> num_points; }
    std::vector<std::vector<float> > depths(num_cams);
    for (unsigned int i = 0; i < num_points; ++i) {
        if (!std::getline(f, line)) break;
        std::istringstream s(line);
        double px, py, pz, cr, cg, cb;
        s >> px >> py >> pz >> cr >> cg >> cb;
        unsigned int nviews = 0;
        s >> nviews;
        for (unsigned int j = 0; j < nviews; ++j) {
            unsigned int cam = 0, sift = 0; float x, y;
            s >> cam >> sift >> x >> y;
            if (!s || cam >= num_cams) { if (error) *error = "malformed measurement list in " + path; return false; }
            cams[cam].worldpoints.push_back(i);
            const double dx = px - cams[cam].C.x, dy = py - cams[cam].C.y, dz = pz - cams[cam].C.z;
            depths[cam].push_back((float)std::sqrt(dx * dx + dy * dy + dz * dz));       // float vector, main_vsfm.cpp:228, 248
        }
    }
    for (unsigned int i = 0; i < num_cams; ++i)
        if (!depths[i].empty()) { std::sort(depths[i].begin(), depths[i].end()); cams[i].median_depth = depths[i][depths[i].size() / 2]; }   // 301-303
    return true;
}

static Vector3d center_of(const Matrix3d& R, const Vector3d& t)      // C = R^T (-t)
{
    return Vector3d(-(R(0, 0) * t.x + R(1, 0) * t.y + R(2, 0) * t.z), -(R(0, 1) * t.x + R(1, 1) * t.y + R(2, 1) * t.z),
                    -(R(0, 2) * t.x + R(1, 2) * t.y + R(2, 2) * t.z));
}
static float median_of(std::vector<float>& d) { if (d.empty()) return 0.0f; std::sort(d.begin(), d.end()); return d[d.size() / 2]; }

bool readBundler(const std::string& bundle_file, const std::string& image_list_file, std::vector<SfMCamera>& cams, std::string* error)
{
    cams.clear();
    std::ifstream f(bundle_file.c_str());
    if (!f) { if (error) *error = "cannot open " + bundle_file; return false; }
    std::string line;
    std::getline(f, line);                       // "# Bundle file v0.3"
    std::getline(f, line);
    unsigned int num_cams = 0, num_points = 0;
    { std::stringstream s(line); s >> num_cams >> num_points; }
    if (num_cams == 0 || num_points == 0) { if (error) *error = "No cameras and/or points in bundle file!"; return false; }   // main_bundler.cpp:159-163
    cams.resize(num_cams);
    for (unsigned int i = 0; i < num_cams; ++i) {
        SfMCamera& c = cams[i];
        c.id = i; c.has_K = false; std::memset(c.K.m, 0, sizeof(c.K.m)); c.median_depth = 0.0f;
        double focal = 0, d1 = 0, d2 = 0;
        bool good = (bool)std::getline(f, line);
        if (good) { std::stringstream s(line); good = (bool)(s >> focal >> d1 >> d2); }
        c.focal = (float)focal;
        c.radial[0] = (float)d1; c.radial[1] = (float)d2; c.radial[2] = 0.0; c.tangential[0] = c.tangential[1] = 0.0;   // float pair, main_bundler.cpp:170, 183
        for (int j = 0; j < 3 && good; ++j) { good = (bool)std::getline(f, line); std::stringstream s(line); good = good && (bool)(s >> c.R(j, 0) >> c.R(j, 1) >> c.R(j, 2)); }
        for (int k = 0; k < 3; ++k) { c.R(1, k) *= -1.0; c.R(2, k) *= -1.0; }                                           // main_bundler.cpp:196-198
        good = good && (bool)std::getline(f, line);
        if (good) { std::stringstream s(line); good = (bool)(s >> c.t.x >> c.t.y >> c.t.z); }
        if (!good) { if (error) *error = "truncated or malformed camera " + std::to_string(i) + " in " + bundle_file; return false; }
        c.t.y *= -1.0; c.t.z *= -1.0;                                                                                    // main_bundler.cpp:210-212
        c.C = center_of(c.R, c.t);
    }
    std::vector<std::vector<float> > depths(num_cams);
    for (unsigned int i = 0; i < num_points; ++i) {
        if (!std::getline(f, line)) break;
        double px = 0, py = 0, pz = 0;
        { std::istringstream s(line); s >> px >> py >> pz; }
        std::getline(f, line);                   // colour
        std::getline(f, line);                   // view list
        std::istringstream s(line);
        unsigned int nviews = 0;
        s >> nviews;
        for (unsigned int j = 0; j < nviews; ++j) {
            unsigned int cam = 0, sift = 0; float x, y;
            s >> cam >> sift >> x >> y;
            if (!s || cam >= num_cams) { if (error) *error = "malformed view list in " + bundle_file; return false; }
            cams[cam].worldpoints.push_back(i);
            const double dx = px - cams[cam].C.x, dy = py - cams[cam].C.y, dz = pz - cams[cam].C.z;
            depths[cam].push_back((float)std::sqrt(dx * dx + dy * dy + dz * dz));
        }
    }
    for (unsigned int i = 0; i < num_cams; ++i) cams[i].median_depth = median_of(depths[i]);
    if (!image_list_file.empty()) {              // main_bundler.cpp:264-286: the first token of line i names image i
        std::ifstream l(image_list_file.c_str());
        unsigned int id = 0;
        while (std::getline(l, line)) {
            std::stringstream s(line);
            std::string fname;
            s >> fname;
            if (!fname.empty() && id < num_cams) cams[id].image = fname;
            ++id;
        }
    }
    return true;
}

// COLMAP's camera models (colmap/sensor/models.h): name, model_id, number of parameters.  `lens` 0: not undistortable here (rejected),
// 1: radtan, 2: fisheye.
struct ColmapModel { const char* name; int id, num_params, lens; };
static const ColmapModel kColmapModels[] = {
    {"SIMPLE_PINHOLE", 0, 3, 1}, {"PINHOLE", 1, 4, 1}, {"SIMPLE_RADIAL", 2, 4, 1}, {"RADIAL", 3, 5, 1}, {"OPENCV", 4, 8, 1},
    {"OPENCV_FISHEYE", 5, 8, 2}, {"FULL_OPENCV", 6, 12, 1}, {"FOV", 7, 5, 0}, {"SIMPLE_RADIAL_FISHEYE", 8, 4, 2}, {"RADIAL_FISHEYE", 9, 5, 2},
    {"THIN_PRISM_FISHEYE", 10, 12, 0}, {"RAD_TAN_THIN_PRISM_FISHEYE", 11, 16, 0},
};

struct ColmapIntr { Matrix3d K; double radial[3], tangential[2]; LensDistortion lens; };

// K, the radial / tangential pair of main_colmap.cpp:160-234 and the full lens of one camera from its parameters in COLMAP's order
static bool colmap_intrinsics(const ColmapModel* m, const std::string& model, unsigned int cam, const double* q, bool want_lens, ColmapIntr& in,
                              std::string* error)
{
    if (!m || m->lens == 0) { if (error) *error = "camera model " + model + " unknown! (camera " + std::to_string(cam) + ")"; return false; }
    if (m->lens == 2 && !want_lens) {
        if (error) *error = "camera " + std::to_string(cam) + " uses the fisheye model " + model + ": its distortion has no place in radial / tangential, "
                            "read the model with the lenses argument of readColmap";
        return false;
    }
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
    std::memset(in.K.m, 0, sizeof(in.K.m));
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
    bool fail(const std::string& why) { if (error) *error = path + ": " + why; return false; }
    bool open()
    {
        std::ifstream f(path.c_str(), std::ios::binary);
        if (!f) return fail("cannot open");
        b.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
        return true;
    }
    template <class T> bool get(T& v, const char* what)
    {
        if (b.size() - pos < sizeof(T)) return fail(std::string("truncated at byte ") + std::to_string(pos) + " (" + what + ")");
        std::memcpy(&v, b.data() + pos, sizeof(T)); pos += sizeof(T);
        return true;
    }
    bool skip(size_t n, const char* what)
    {
        if (b.size() - pos < n) return fail(std::string("truncated at byte ") + std::to_string(pos) + " (" + what + ")");
        pos += n;
        return true;
    }
    // a record count: each record takes at least min_bytes, so a count the rest of the file cannot hold is malformed
    bool count(uint64_t& n, size_t min_bytes, const char* what)
    {
        if (!get(n, what)) return false;
        if (n > (b.size() - pos) / min_bytes) return fail(std::string(what) + " " + std::to_string(n) + " exceeds what the file holds");
        return true;
    }
    bool name(std::string& s)
    {
        const void* z = std::memchr(b.data() + pos, 0, b.size() - pos);
        if (!z) return fail("unterminated image name at byte " + std::to_string(pos));
        const size_t n = (const unsigned char*)z - (b.data() + pos);
        s.assign((const char*)b.data() + pos, n); pos += n + 1;
        return true;
    }
    bool id32(uint64_t v, unsigned int& out, const char* what)
    {
        if (v > 0xFFFFFFFFull) return fail(std::string(what) + " " + std::to_string(v) + " does not fit unsigned int");
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
    if (!text && !binary) { if (error) *error = "at least one of the colmap result files does not exist in sfm folder: " + folder; return false; }
    std::map<unsigned int, ColmapIntr> intr;
    std::map<unsigned int, Vector3d> wps;        // world points referenced by a kept image; (0,0,0) until points3D fills them in
    // one image of images.txt / .bin: kept (and its camera's lens recorded) when its camera is known
    auto add_image = [&](unsigned int img, double qw, double qx, double qy, double qz, double tx, double ty, double tz, unsigned int cam,
                         const std::string& name) {
        std::map<unsigned int, ColmapIntr>::const_iterator it = intr.find(cam);
        if (it == intr.end()) return false;
        SfMCamera c;
        c.id = img; c.image = name; c.has_K = true; c.K = it->second.K; c.focal = 0.0f; c.median_depth = 0.0f;
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
            ColmapIntr in;
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
            if (!m) return fc.fail("camera model id " + std::to_string(mid) + " of camera " + std::to_string(cam) + " unknown!");
            double q[16] = {0};
            for (int k = 0; k < m->num_params; ++k) if (!fc.get(q[k], "camera parameters")) return false;
            ColmapIntr in;
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
    for (size_t i = 0; i < cams.size(); ++i) {   // main_colmap.cpp:386-401
        std::vector<float> d;
        for (unsigned int w : cams[i].worldpoints) {
            const Vector3d& P = wps[w];
            const double dx = cams[i].C.x - P.x, dy = cams[i].C.y - P.y, dz = cams[i].C.z - P.z;
            d.push_back((float)std::sqrt(dx * dx + dy * dy + dz * dz));
        }
        cams[i].median_depth = median_of(d);
    }
    if (cams.empty()) { if (lenses) lenses->clear(); if (error) *error = "no usable image in " + folder; return false; }
    return true;
}

Matrix3d intrinsicsFromFocal(float focal, int w, int h)
{
    Matrix3d K; std::memset(K.m, 0, sizeof(K.m));
    K(0, 0) = focal; K(1, 1) = focal; K(0, 2) = float(w) / 2.0f; K(1, 2) = float(h) / 2.0f; K(2, 2) = 1.0;
    return K;
}

}  // namespace L3DPP

// C wrapper (include/l3dpp_capi.h): flat arrays
extern "C" {
void* l3dpp_nvm_open(const char* path, char* err, int errcap)
{
    std::vector<L3DPP::NVMCamera>* v = new std::vector<L3DPP::NVMCamera>();
    std::string e;
    if (!L3DPP::readNVM(path, *v, &e)) { l3dpp_copy_str(e, err, errcap); delete v; return nullptr; }
    return v;
}
void l3dpp_nvm_close(void* h) { delete (std::vector<L3DPP::NVMCamera>*)h; }
int l3dpp_nvm_num_cameras(void* h) { return (int)((std::vector<L3DPP::NVMCamera>*)h)->size(); }
int l3dpp_nvm_camera(void* h, int i, double* R9, double* t3, double* C3, float* focal, float* distortion, float* median_depth, int* num_wps, char* name, int namecap)
{
    const std::vector<L3DPP::NVMCamera>& v = *(std::vector<L3DPP::NVMCamera>*)h;
    if (i < 0 || i >= (int)v.size()) return -1;
    const L3DPP::NVMCamera& c = v[i];
    for (int k = 0; k < 9; ++k) R9[k] = c.R.m[k];
    t3[0] = c.t.x; t3[1] = c.t.y; t3[2] = c.t.z; C3[0] = c.C.x; C3[1] = c.C.y; C3[2] = c.C.z;
    *focal = c.focal; *distortion = c.distortion; *median_depth = c.median_depth; *num_wps = (int)c.worldpoints.size();
    l3dpp_copy_str(c.image, name, namecap);
    return 0;
}
int l3dpp_nvm_worldpoints(void* h, int i, unsigned int* out, int cap)
{
    const std::vector<L3DPP::NVMCamera>& v = *(std::vector<L3DPP::NVMCamera>*)h;
    if (i < 0 || i >= (int)v.size()) return -1;
    int n = 0;
    for (unsigned int w : v[i].worldpoints) { if (n < cap) out[n] = w; ++n; }
    return n;
}
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
    const std::vector<L3DPP::LensDistortion>& v = ((L3DSfMHandle*)h)->lenses;
    if (i < 0 || i >= (int)v.size()) return -1;
    lens9[0] = v[i].model;
    for (int k = 0; k < 6; ++k) lens9[1 + k] = v[i].k[k];
    lens9[7] = v[i].p[0]; lens9[8] = v[i].p[1];
    return 0;
}
int l3dpp_sfm_camera(void* h, int i, double* head5, double* K9, double* R9, double* t3, double* C3, double* dist5, char* name, int namecap)
{
    const std::vector<L3DPP::SfMCamera>& v = ((L3DSfMHandle*)h)->cams;
    if (i < 0 || i >= (int)v.size()) return -1;
    const L3DPP::SfMCamera& c = v[i];
    head5[0] = c.id; head5[1] = c.has_K; head5[2] = c.focal; head5[3] = c.median_depth; head5[4] = (double)c.worldpoints.size();
    for (int k = 0; k < 9; ++k) { K9[k] = c.K.m[k]; R9[k] = c.R.m[k]; }
    t3[0] = c.t.x; t3[1] = c.t.y; t3[2] = c.t.z; C3[0] = c.C.x; C3[1] = c.C.y; C3[2] = c.C.z;
    for (int k = 0; k < 3; ++k) dist5[k] = c.radial[k];
    dist5[3] = c.tangential[0]; dist5[4] = c.tangential[1];
    l3dpp_copy_str(c.image, name, namecap);
    return 0;
}
int l3dpp_sfm_worldpoints(void* h, int i, unsigned int* out, int cap)
{
    const std::vector<L3DPP::SfMCamera>& v = ((L3DSfMHandle*)h)->cams;
    if (i < 0 || i >= (int)v.size()) return -1;
    int n = 0;
    for (unsigned int w : v[i].worldpoints) { if (n < cap) out[n] = w; ++n; }
    return n;
}
void l3dpp_intrinsics_from_focal(float focal, int w, int h, double* K9) { const L3DPP::Matrix3d K = L3DPP::intrinsicsFromFocal(focal, w, h); for (int k = 0; k < 9; ++k) K9[k] = K.m[k]; }
}
