// line3d_bin.cc — the reference's two binary files without Boost: the result file of save3DLinesAsBIN (line3D.cc:2690-2711) and
// the per-view segment cache (line3D.cc:295-309, 363-366).  Both are boost::archive::binary_oarchive files (serialization.h:38-46);
// this file reads and writes exactly the types they hold, in the order of the reference's serialize() methods.  Byte layout:
// DESIGN.md §6a.  Host only.
#include "../../include/line3d_io.h"
#include "../../include/l3dpp_capi.h"
#include "l3dpp_wrap.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <iterator>
#include <sstream>

namespace L3DPP {
namespace {

const char SIGNATURE[] = "serialization::archive";          // 22 characters, stored after its u64 length
const uint16_t LIBRARY_VERSION = 10;                        // what the reference's result files carry
const uint16_t MIN_LIBRARY_VERSION = 8;                     // older archives store class versions and counts in other widths
const unsigned char TYPE_SIZES[4] = {4, 8, 4, 8};           // sizeof(int), sizeof(long), sizeof(float), sizeof(double)

// Boost writes an object's class info (tracking flag u8, class version u32) before the FIRST object of each class in the archive;
// primitives carry none.  One flag per class of these files records whether it has been written / read yet.
enum Cls { C_LINES, C_LINE, C_SEG3_LIST, C_SEG3, C_CLUSTER, C_SEG2_LIST, C_SEG2, C_ARRAY, C_FLOAT4, C_COUNT };

class Out {
public:
    Out()
    {
        put<uint64_t>(22); buf_.append(SIGNATURE, 22); put<uint16_t>(LIBRARY_VERSION);
        buf_.append((const char*)TYPE_SIZES, 4); put<int32_t>(1);
    }
    template <class T> void put(T v) { buf_.append((const char*)&v, sizeof(v)); }
    void cls(Cls c) { if (!seen_[c]) { put<uint8_t>(0); put<uint32_t>(0); seen_[c] = true; } }
    void count(uint64_t n) { put<uint64_t>(n); put<uint32_t>(0); }             // collection_size_type + item_version_type
    void seg3(const Segment3D& s)                                                // segment3D.h:99-115
    {
        cls(C_SEG3);
        put<float>(s.length()); put<uint8_t>(s.valid() ? 1 : 0);
        const Vector3d v[3] = {s.P1(), s.P2(), s.dir()};
        for (const Vector3d& p : v) { put<double>(p.x); put<double>(p.y); put<double>(p.z); }
    }
    bool save(const std::string& path, std::string* error) const
    {
        std::ofstream f(path.c_str(), std::ios::binary);
        if (f) f.write(buf_.data(), (std::streamsize)buf_.size());
        if (f) f.close();
        if (!f) { if (error) *error = "cannot open " + path + " for writing"; return false; }
        return true;
    }
private:
    std::string buf_;
    bool seen_[C_COUNT] = {};
};

class In {
public:
    In(const std::string& path) : path_(path) {}
    std::string err;

    bool open()
    {
        std::ifstream f(path_.c_str(), std::ios::binary);
        if (!f) return fail("cannot open");
        buf_.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
        if (f.bad()) return fail("cannot read");
        uint64_t len = 0; uint16_t lib = 0; unsigned char sizes[4]; int32_t one = 0;
        if (!get(len) || len != 22 || !bytes(22) || std::memcmp(&buf_[pos_ - 22], SIGNATURE, 22) != 0)
            return fail("not a Boost binary archive (no \"serialization::archive\" signature)");
        if (!get(lib)) return false;
        if (lib < MIN_LIBRARY_VERSION) return fail("Boost archive library version " + std::to_string(lib) + " is older than the supported 8");
        if (!bytes(4)) return false;
        std::memcpy(sizes, &buf_[pos_ - 4], 4);
        if (std::memcmp(sizes, TYPE_SIZES, 4) != 0) return fail("type sizes of another platform (expected int 4, long 8, float 4, double 8)");
        if (!get(one)) return false;
        if (one != 1) return fail("archive of the other byte order");
        return true;
    }
    template <class T> bool get(T& v)
    {
        if (!bytes(sizeof(T))) return false;
        std::memcpy(&v, &buf_[pos_ - sizeof(T)], sizeof(T));
        return true;
    }
    bool cls(Cls c)
    {
        if (seen_[c]) return true;
        uint8_t tracking = 0; uint32_t version = 0;
        if (!get(tracking) || !get(version)) return false;
        if (tracking != 0 || version != 0) return fail("object tracking or a class version at byte " + std::to_string(pos_ - 5) + " (neither is used by these files)");
        seen_[c] = true;
        return true;
    }
    // a collection count; `item_bytes` is the smallest size one element can have, so a count the rest of the file cannot hold fails here
    bool count(uint64_t& n, uint64_t item_bytes)
    {
        uint32_t item_version = 0;
        if (!get(n) || !get(item_version)) return false;
        if (item_version != 0) return fail("item version " + std::to_string(item_version) + " at byte " + std::to_string(pos_ - 4));
        if (n > remaining() / item_bytes) return fail("count " + std::to_string(n) + " at byte " + std::to_string(pos_ - 12) + " exceeds the remaining bytes");
        return true;
    }
    bool seg3(std::list<Segment3D>& to)                                         // appends the segment read
    {
        float length = 0; uint8_t valid = 0; double d[9];
        if (!cls(C_SEG3) || !get(length) || !get(valid)) return false;
        if (valid > 1) return fail("bool value " + std::to_string(valid) + " at byte " + std::to_string(pos_ - 1));
        for (double& x : d) if (!get(x)) return false;
        to.push_back(Segment3D(Vector3d(d[0], d[1], d[2]), Vector3d(d[3], d[4], d[5]), Vector3d(d[6], d[7], d[8]), length, valid != 0));
        return true;
    }
    bool finish()
    {
        if (pos_ != buf_.size()) return fail(std::to_string(buf_.size() - pos_) + " unexpected bytes after the archive at byte " + std::to_string(pos_));
        return true;
    }
    uint64_t remaining() const { return buf_.size() - pos_; }
    bool fail(const std::string& what) { if (err.empty()) err = path_ + ": " + what; return false; }

private:
    bool bytes(size_t n)
    {
        if (remaining() < n) return fail("truncated at byte " + std::to_string(buf_.size()) + " (" + std::to_string(n) + " more bytes expected at byte " + std::to_string(pos_) + ")");
        pos_ += n;
        return true;
    }
    std::string path_, buf_;
    size_t pos_ = 0;
    bool seen_[C_COUNT] = {};
};

const uint64_t SEG3_BYTES = 4 + 1 + 9 * 8;                          // length, valid, P1, P2, dir
const uint64_t SEG2_BYTES = 2 * 4;                                  // camID, segID
const uint64_t LINE_BYTES = 12 + SEG3_BYTES + 12 + 4;               // empty segment list, cluster line, empty residual list, ref view

bool reject(std::string* error, const std::string& what) { if (error) *error = what; return false; }

}  // namespace

bool read3DLinesBIN(const std::string& path, std::vector<FinalLine3D>& lines, std::string* error)
{
    lines.clear();
    In in(path);
    std::vector<FinalLine3D> out;
    uint64_t n = 0;
    bool ok = in.open() && in.cls(C_LINES) && in.count(n, LINE_BYTES);
    for (uint64_t i = 0; ok && i < n; ++i) {                                       // FinalLine3D, segment3D.h:173-177
        std::list<Segment3D> segs;
        uint64_t ns = 0;
        ok = in.cls(C_LINE) && in.cls(C_SEG3_LIST) && in.count(ns, SEG3_BYTES);
        for (uint64_t k = 0; ok && k < ns; ++k) ok = in.seg3(segs);
        std::list<Segment3D> line;                                                  // LineCluster3D, segment3D.h:155-160
        std::list<Segment2D> res;
        uint64_t nr = 0;
        ok = ok && in.cls(C_CLUSTER) && in.seg3(line) && in.cls(C_SEG2_LIST) && in.count(nr, SEG2_BYTES);
        for (uint64_t k = 0; ok && k < nr; ++k) {                                   // Segment2D, commons.h:126-130
            uint32_t cam = 0, seg = 0;
            ok = in.cls(C_SEG2) && in.get(cam) && in.get(seg);
            if (ok) res.push_back(Segment2D(cam, seg));
        }
        uint32_t ref_view = 0;
        ok = ok && in.get(ref_view);
        if (ok) out.push_back(FinalLine3D{segs, LineCluster3D(line.front(), res, ref_view)});
    }
    if (!(ok && in.finish())) return reject(error, in.err);
    lines.swap(out);
    return true;
}

bool write3DLinesBIN(const std::string& path, const std::vector<FinalLine3D>& lines, std::string* error)
{
    Out o;
    o.cls(C_LINES);
    o.count(lines.size());
    for (const FinalLine3D& L : lines) {
        o.cls(C_LINE);
        o.cls(C_SEG3_LIST);
        o.count(L.collinear3Dsegments_.size());
        for (const Segment3D& s : L.collinear3Dsegments_) o.seg3(s);
        const LineCluster3D& c = L.underlyingCluster_;
        o.cls(C_CLUSTER);
        o.seg3(c.seg3D());
        o.cls(C_SEG2_LIST);
        o.count(c.residuals()->size());
        for (const Segment2D& r : *c.residuals()) { o.cls(C_SEG2); o.put<uint32_t>(r.camID()); o.put<uint32_t>(r.segID()); }
        o.put<uint32_t>(c.reference_view());
    }
    return o.save(path, error);
}

// DataArray<float4> (dataArray.h:355-374): width_, height_, real_width_ (u32), pitchCPU_, strideCPU_, pitchGPU_, strideGPU_ (size_t),
// then real_width_ * height_ float4 (dataArray.h:64-70: x, y, z, w).  Rows are padded to 32 bytes (dataArray.h:104-125); the cache
// holds one row and View reads its first width_ entries.
bool readSegmentCache(const std::string& path, std::vector<Vec4f>& segments, std::string* error)
{
    segments.clear();
    In in(path);
    uint32_t width = 0, height = 0, real_width = 0;
    uint64_t pitch = 0, stride = 0, pitch_gpu = 0, stride_gpu = 0;
    if (!(in.open() && in.cls(C_ARRAY) && in.get(width) && in.get(height) && in.get(real_width) && in.get(pitch) && in.get(stride) &&
          in.get(pitch_gpu) && in.get(stride_gpu)))
        return reject(error, in.err);
    if (height != 1 || real_width < width || stride != real_width || pitch != 16ull * real_width)
        return reject(error, path + ": not a segment cache (width " + std::to_string(width) + ", height " + std::to_string(height) +
                                 ", real width " + std::to_string(real_width) + ", stride " + std::to_string(stride) + ", pitch " + std::to_string(pitch) + ")");
    if (real_width > in.remaining() / 16) return reject(error, path + ": " + std::to_string(real_width) + " segments exceed the remaining bytes");
    std::vector<Vec4f> out;
    out.reserve(width);
    bool ok = real_width == 0 || in.cls(C_FLOAT4);
    for (uint32_t i = 0; ok && i < real_width; ++i) {
        Vec4f v;
        for (int k = 0; ok && k < 4; ++k) ok = in.get(v.v[k]);
        if (ok && i < width) out.push_back(v);
    }
    if (!(ok && in.finish())) return reject(error, in.err);
    segments.swap(out);
    return true;
}

bool writeSegmentCache(const std::string& path, const std::vector<Vec4f>& segments, std::string* error)
{
    if (segments.size() > 0x7fffffffu) return reject(error, path + ": too many segments for a DataArray");
    const uint32_t width = (uint32_t)segments.size();
    const uint32_t real_width = width + ((16ull * width) % 32 ? 1 : 0);          // dataArray.h:111-122 for 16-byte elements
    Out o;
    o.cls(C_ARRAY);
    o.put<uint32_t>(width); o.put<uint32_t>(1); o.put<uint32_t>(real_width);
    o.put<uint64_t>(16ull * real_width); o.put<uint64_t>(real_width); o.put<uint64_t>(0); o.put<uint64_t>(0);   // never on the GPU when stored
    if (real_width) o.cls(C_FLOAT4);
    for (uint32_t i = 0; i < real_width; ++i)
        for (int k = 0; k < 4; ++k) o.put<float>(i < width ? segments[i].v[k] : 0.0f);
    return o.save(path, error);
}

bool preparedImageSize(int w, int h, int max_img_width, int& out_w, int& out_h, float* scale)
{
    out_w = w; out_h = h;
    if (scale) *scale = 1.0f;
    const int max_dim = std::max(w, h);
    if (!(max_img_width > 0 && max_dim > max_img_width)) return false;
    // cv::resize(img, out, Size(), s, s): Size(saturate_cast<int>(cols * s), saturate_cast<int>(rows * s)) in double, rounded to nearest even
    const float s = float(max_img_width) / float(max_dim);
    out_w = (int)std::llrint((double)w * (double)s);
    out_h = (int)std::llrint((double)h * (double)s);
    if (scale) *scale = s;
    return true;
}

std::string segmentCachePath(const std::string& output_folder, unsigned int camID, int w, int h, int max_img_width)
{
    int nw, nh;
    preparedImageSize(w, h, max_img_width, nw, nh);
    std::stringstream p;
    p << output_folder << "/L3D++_data/segments_L3D++_" << camID << "_" << nw << "x" << nh << "_" << L3D_DEF_MAX_NUM_SEGMENTS << ".bin";
    return p.str();
}

}  // namespace L3DPP

// C wrapper (include/l3dpp_capi.h), handles like l3dpp_nvm_*.  No GPU is involved.
extern "C" {
static void l3dpp_seg_out(const L3DPP::Segment3D& s, int line, l3dpp_bin_seg& o)
{
    o.line = line; o.valid = s.valid() ? 1 : 0; o.length = s.length(); o.pad = 0;
    const L3DPP::Vector3d v[3] = {s.P1(), s.P2(), s.dir()};
    double* d[3] = {o.p1, o.p2, o.dir};
    for (int k = 0; k < 3; ++k) { d[k][0] = v[k].x; d[k][1] = v[k].y; d[k][2] = v[k].z; }
}
static L3DPP::Segment3D l3dpp_seg_in(const l3dpp_bin_seg& o)
{
    return L3DPP::Segment3D(L3DPP::Vector3d(o.p1[0], o.p1[1], o.p1[2]), L3DPP::Vector3d(o.p2[0], o.p2[1], o.p2[2]),
                            L3DPP::Vector3d(o.dir[0], o.dir[1], o.dir[2]), o.length, o.valid != 0);
}

void* l3dpp_bin_open(const char* path, char* err, int errcap)
{
    std::vector<L3DPP::FinalLine3D>* v = new std::vector<L3DPP::FinalLine3D>();
    std::string e;
    if (!L3DPP::read3DLinesBIN(path, *v, &e)) { l3dpp_copy_str(e, err, errcap); delete v; return nullptr; }
    return v;
}
void l3dpp_bin_close(void* h) { delete (std::vector<L3DPP::FinalLine3D>*)h; }
void l3dpp_bin_sizes(void* h, long long* nlines, long long* nsegs, long long* nres)
{
    const std::vector<L3DPP::FinalLine3D>& v = *(std::vector<L3DPP::FinalLine3D>*)h;
    *nlines = (long long)v.size(); *nsegs = *nres = 0;
    for (const L3DPP::FinalLine3D& L : v) { *nsegs += (long long)L.collinear3Dsegments_.size(); *nres += (long long)L.underlyingCluster_.size(); }
}
void l3dpp_bin_get(void* h, l3dpp_bin_line* lines, l3dpp_bin_seg* clusters, l3dpp_bin_seg* segs, l3dpp_bin_res* res)
{
    const std::vector<L3DPP::FinalLine3D>& v = *(std::vector<L3DPP::FinalLine3D>*)h;
    size_t so = 0, ro = 0;
    for (size_t i = 0; i < v.size(); ++i) {
        const L3DPP::FinalLine3D& L = v[i];
        lines[i].nseg = (int)L.collinear3Dsegments_.size(); lines[i].nres = (int)L.underlyingCluster_.size();
        lines[i].reference_view = L.underlyingCluster_.reference_view(); lines[i].pad = 0;
        l3dpp_seg_out(L.underlyingCluster_.seg3D(), (int)i, clusters[i]);
        for (const L3DPP::Segment3D& s : L.collinear3Dsegments_) l3dpp_seg_out(s, (int)i, segs[so++]);
        for (const L3DPP::Segment2D& r : *L.underlyingCluster_.residuals()) { res[ro].line = (int)i; res[ro].cam = r.camID(); res[ro].seg = r.segID(); ++ro; }
    }
}
int l3dpp_bin_write(const char* path, long long nlines, const l3dpp_bin_line* lines, const l3dpp_bin_seg* clusters, const l3dpp_bin_seg* segs,
                    const l3dpp_bin_res* res, char* err, int errcap)
{
    std::vector<L3DPP::FinalLine3D> v;
    size_t so = 0, ro = 0;
    for (long long i = 0; i < nlines; ++i) {
        if (lines[i].nseg < 0 || lines[i].nres < 0) { l3dpp_copy_str("negative segment or residual count", err, errcap); return -1; }
        std::list<L3DPP::Segment3D> s;
        for (int k = 0; k < lines[i].nseg; ++k) s.push_back(l3dpp_seg_in(segs[so++]));
        std::list<L3DPP::Segment2D> r;
        for (int k = 0; k < lines[i].nres; ++k, ++ro) r.push_back(L3DPP::Segment2D(res[ro].cam, res[ro].seg));
        v.push_back(L3DPP::FinalLine3D{s, L3DPP::LineCluster3D(l3dpp_seg_in(clusters[i]), r, lines[i].reference_view)});
    }
    std::string e;
    if (!L3DPP::write3DLinesBIN(path, v, &e)) { l3dpp_copy_str(e, err, errcap); return -1; }
    return 0;
}

void* l3dpp_segcache_open(const char* path, char* err, int errcap)
{
    std::vector<L3DPP::Vec4f>* v = new std::vector<L3DPP::Vec4f>();
    std::string e;
    if (!L3DPP::readSegmentCache(path, *v, &e)) { l3dpp_copy_str(e, err, errcap); delete v; return nullptr; }
    return v;
}
void l3dpp_segcache_close(void* h) { delete (std::vector<L3DPP::Vec4f>*)h; }
long long l3dpp_segcache_count(void* h) { return (long long)((std::vector<L3DPP::Vec4f>*)h)->size(); }
void l3dpp_segcache_get(void* h, float* xy4)
{
    const std::vector<L3DPP::Vec4f>& v = *(std::vector<L3DPP::Vec4f>*)h;
    if (!v.empty()) std::memcpy(xy4, v.data(), v.size() * sizeof(L3DPP::Vec4f));
}
int l3dpp_segcache_write(const char* path, const float* xy4, long long n, char* err, int errcap)
{
    if (n < 0) { l3dpp_copy_str("negative segment count", err, errcap); return -1; }
    std::vector<L3DPP::Vec4f> v((size_t)n);
    if (n) std::memcpy(v.data(), xy4, (size_t)n * sizeof(L3DPP::Vec4f));
    std::string e;
    if (!L3DPP::writeSegmentCache(path, v, &e)) { l3dpp_copy_str(e, err, errcap); return -1; }
    return 0;
}
int l3dpp_segcache_path(const char* folder, unsigned int cam, int w, int h, int max_img_width, char* buf, int cap)
{
    const std::string s = L3DPP::segmentCachePath(folder, cam, w, h, max_img_width);
    if ((int)s.size() + 1 > cap) return -1;
    std::memcpy(buf, s.c_str(), s.size() + 1);
    return (int)s.size();
}
}
