// line3d_host.cc — host side of L3DPP::Line3D (include/line3d.h) on top of the C ABI (include/l3d_capi.h).
//
// What stays on the host is what line3D.cc does around its accelerator calls: camera algebra (View::View, view.cc:6-42),
// translate / untranslate (line3D.cc:500-575), spatial regulariser k (view.cc:301-314), visual neighbours
// (line3D.cc:578-699), the view-pair list and fundamental matrices (702-741, 861-897), then after the device stages the
// "unused"/local-id bookkeeping of the affinity matrix (1881-1900, 1982-2023), the symmetrisation after diffusion
// (2036-2071), graph clustering (clustering.cc:6-48) and the cluster -> 3D segment tail (2079-2452) + writers.
// All matching / scoring / affinity / diffusion arithmetic runs on the GPU; without a GPU the constructor fails.
#include "../../include/line3d.h"
#include "../../include/line3d_io.h"   // segment cache + .bin writer (csrc/line3d_bin.cc)
#include <nvtx3/nvToolsExt.h>      // header-only; ranges show up in nsys / ncu timelines
#include "../../include/l3d_capi.h"
#include "../../include/l3dpp_capi.h"
#include "l3d_pose_select.h"
#include <cuda_runtime_api.h>          // cudaGetDevice: undistortImage runs on the caller's current device

#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <mutex>
#include <queue>
#include <set>
#include <sstream>
#include <stdexcept>
#include <thread>
#include <type_traits>
#include <sys/stat.h>                  // mkdir: the segment cache's folder

namespace L3DPP {

// Independent per-cluster host work (the reference runs the same loops under `#pragma omp parallel for`, line3D.cc:2125, 2283):
// static partition over a few std::threads, results stored by index, so the output order does not depend on timing.
template <class F> static void parallel_for(size_t n, F&& body)
{
    unsigned int nt = std::min<unsigned int>(std::max(1u, std::thread::hardware_concurrency()), 32u);
    if (const char* e = getenv("L3D_HOST_THREADS")) nt = (unsigned int)std::max(1, atoi(e));
    if (n < 256 || nt <= 1) { for (size_t i = 0; i < n; ++i) body(i); return; }
    nt = (unsigned int)std::min<size_t>(nt, n / 64);
    std::vector<std::thread> th;
    for (unsigned int t = 0; t < nt; ++t)
        th.emplace_back([&, t]() { for (size_t i = n * t / nt; i < n * (t + 1) / nt; ++i) body(i); });
    for (auto& x : th) x.join();
}


namespace {
const double EPS = 1e-12;                    // L3D_EPS commons.h:92
const float MIN_SIMILARITY_3D = 0.50f, MIN_BEST_SCORE_3D = 0.75f, MIN_BEST_SCORE_PERC = 0.10f, MIN_AFFINITY = 0.50f;   // commons.h:58-60,68
const int RDD_MAX_ITER = 10;                 // commons.h:65

inline Vector3d operator+(const Vector3d& a, const Vector3d& b) { return Vector3d(a.x + b.x, a.y + b.y, a.z + b.z); }
inline Vector3d operator-(const Vector3d& a, const Vector3d& b) { return Vector3d(a.x - b.x, a.y - b.y, a.z - b.z); }
inline Vector3d operator*(const Vector3d& a, double s) { return Vector3d(a.x * s, a.y * s, a.z * s); }
inline double dot(const Vector3d& a, const Vector3d& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline double norm(const Vector3d& a) { return std::sqrt(dot(a, a)); }
inline Vector3d unit(const Vector3d& a) { double n2 = dot(a, a); if (n2 > 0) { double n = std::sqrt(n2); return Vector3d(a.x / n, a.y / n, a.z / n); } return a; }
inline Matrix3d matmul(const Matrix3d& a, const Matrix3d& b)
{ Matrix3d r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += a(i, k) * b(k, j); r(i, j) = s; } return r; }
inline Vector3d matvec(const Matrix3d& a, const Vector3d& v)
{ return Vector3d(a(0, 0) * v.x + a(0, 1) * v.y + a(0, 2) * v.z, a(1, 0) * v.x + a(1, 1) * v.y + a(1, 2) * v.z, a(2, 0) * v.x + a(2, 1) * v.y + a(2, 2) * v.z); }
template <class T> T median_of(std::vector<T>& v, T if_empty)   // sorts v; the reference's median is the element at size / 2
{ if (v.empty()) return if_empty; std::sort(v.begin(), v.end()); return v[v.size() / 2]; }
inline Matrix3d transposed(const Matrix3d& a) { Matrix3d r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r(i, j) = a(j, i); return r; }
Matrix3d inverted(const Matrix3d& a)   // adjugate / determinant
{
    Matrix3d r;
    const double c00 = a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1), c01 = a(1, 2) * a(2, 0) - a(1, 0) * a(2, 2), c02 = a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0);
    const double id = 1.0 / (a(0, 0) * c00 + a(0, 1) * c01 + a(0, 2) * c02);
    r(0, 0) = c00 * id; r(1, 0) = c01 * id; r(2, 0) = c02 * id;
    r(0, 1) = (a(0, 2) * a(2, 1) - a(0, 1) * a(2, 2)) * id; r(1, 1) = (a(0, 0) * a(2, 2) - a(0, 2) * a(2, 0)) * id; r(2, 1) = (a(0, 1) * a(2, 0) - a(0, 0) * a(2, 1)) * id;
    r(0, 2) = (a(0, 1) * a(1, 2) - a(0, 2) * a(1, 1)) * id; r(1, 2) = (a(0, 2) * a(1, 0) - a(0, 0) * a(1, 2)) * id; r(2, 2) = (a(0, 0) * a(1, 1) - a(0, 1) * a(1, 0)) * id;
    return r;
}

struct HostView {
    unsigned int id = 0;
    int width = 0, height = 0;
    Matrix3d K, R, RtKinv;
    Vector3d t, C, pp;
    float C_f3[3], RtKinv_f[9];      // frozen at construction like view.cc:35-40 (NOT updated by translate)
    float k = 0.f, median_depth = 0.f, min_line_length = 0.f;
    std::vector<Vec4f> lines;
    std::list<unsigned int> wps_or_neighbors;
    long long seg_off = 0;           // global segment index of segment 0 (views in ascending camID)

    Vector3d ray(double x, double y) const { return unit(matvec(RtKinv, Vector3d(x, y, 1.0))); }
    void shift(const Vector3d& d) { C = C + d; t = matvec(R, C) * -1.0; }             // View::translate view.cc:510-514
    void project(const Vector3d& P, double& u, double& v) const                       // View::project view.cc:374-393
    {
        Vector3d q = matvec(R, P) + t;
        const double xn = (1.0 * q.x + 0.0 * q.z) / q.z, yn = (1.0 * q.y + 0.0 * q.z) / q.z;
        Vector3d h = matvec(K, Vector3d(xn, yn, 1));
        u = h.x / h.z; v = h.y / h.z;
    }
};

struct Affinity { std::vector<int> i, j; std::vector<float> w; };   // the CLEdges (clustering.h:47-51) as l3d_affinity_matrix fills them

// Felzenszwalb-Huttenlocher graph segmentation as used by the reference (clustering.cc:6-48, universe.h:49-104):
// edges visited by ascending weight (stable), components merge while w <= both thresholds, threshold = w + c/|C|.
class DisjointSets {
public:
    explicit DisjointSets(int n) : parent_(n), rank_(n, 0), size_(n, 1) { for (int i = 0; i < n; ++i) parent_[i] = i; }
    int find(int x) { int root = x; while (root != parent_[root]) root = parent_[root]; parent_[x] = root; return root; }   // single-step compression like universe.h:70-78
    int unite(int a, int b)
    {
        if (rank_[a] > rank_[b]) { parent_[b] = a; size_[a] += size_[b]; return a; }
        parent_[a] = b; size_[b] += size_[a];
        if (rank_[a] == rank_[b]) ++rank_[b];
        return b;
    }
    int size(int x) const { return size_[x]; }
private:
    std::vector<int> parent_, rank_, size_;
};

// `order` (optional): indices of the edges by ascending weight, ties in list order (from l3d_argsort_f32 for big lists)
std::vector<int> segment_graph(const Affinity& A, int n, float c, const std::vector<unsigned int>* order)
{
    std::vector<unsigned int> local;
    if (!order) {
        local.resize(A.w.size());
        for (size_t i = 0; i < local.size(); ++i) local[i] = (unsigned int)i;
        std::stable_sort(local.begin(), local.end(), [&](unsigned int a, unsigned int b) { return A.w[a] < A.w[b]; });
        order = &local;
    }
    DisjointSets u(n);
    std::vector<float> thr(n, c);
    for (unsigned int idx : *order) {
        const float w = A.w[idx];
        int a = u.find(A.i[idx]), b = u.find(A.j[idx]);
        if (a == b || !(w <= thr[a] && w <= thr[b])) continue;
        u.unite(a, b);
        a = u.find(a);
        thr[a] = w + c / (float)u.size(a);
    }
    std::vector<int> label(n);
    for (int i = 0; i < n; ++i) label[i] = u.find(i);
    return label;
}

// dominant eigenvector of a symmetric positive semi-definite 3x3 matrix by cyclic Jacobi rotations; plays the role of
// the JacobiSVD of the scatter matrix in get3DlineFromCluster (line3D.cc:2196-2211)
Vector3d principal_axis(double A[3][3])
{
    double Q[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 60; ++sweep) {
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        if (off < 1e-300) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (std::fabs(A[p][q]) < 1e-300) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
                const double tt = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                const double cs = 1.0 / std::sqrt(tt * tt + 1.0), sn = tt * cs;
                for (int k = 0; k < 3; ++k) { const double x = A[k][p], y = A[k][q]; A[k][p] = cs * x - sn * y; A[k][q] = sn * x + cs * y; }
                for (int k = 0; k < 3; ++k) { const double x = A[p][k], y = A[q][k]; A[p][k] = cs * x - sn * y; A[q][k] = sn * x + cs * y; }
                for (int k = 0; k < 3; ++k) { const double x = Q[k][p], y = Q[k][q]; Q[k][p] = cs * x - sn * y; Q[k][q] = sn * x + cs * y; }
            }
    }
    int m = 0;
    if (A[1][1] > A[m][m]) m = 1;
    if (A[2][2] > A[m][m]) m = 2;
    return unit(Vector3d(Q[0][m], Q[1][m], Q[2][m]));
}
}  // namespace

// ------------------------------------------------------------------------------------------------ Segment3D
Segment3D::Segment3D() : P1_(0, 0, 0), P2_(0, 0, 0), dir_(0, 0, 0), length_(0.0f), valid_(false) {}
Segment3D::Segment3D(const Vector3d& P1, const Vector3d& P2)
{
    length_ = (float)norm(P1 - P2);
    if (length_ > EPS) { P1_ = P1; P2_ = P2; dir_ = unit(P2 - P1); valid_ = true; }
    else { P1_ = P2_ = dir_ = Vector3d(0, 0, 0); length_ = 0.0f; valid_ = false; }
}
float Segment3D::distance_Point2Line(const Vector3d& P) const
{
    const Vector3d w = P - P1_;
    const double d[3] = {dir_.x, dir_.y, dir_.z}, ww[3] = {w.x, w.y, w.z};
    double h[3];
    for (int i = 0; i < 3; ++i) h[i] = (d[i] * ww[0]) * d[0] + (d[i] * ww[1]) * d[1] + (d[i] * ww[2]) * d[2];
    return (float)norm(Vector3d(P1_.x + h[0], P1_.y + h[1], P1_.z + h[2]) - P);
}
void Segment3D::translate(const Vector3d& t) { P1_ = P1_ + t; P2_ = P2_ + t; }

// ------------------------------------------------------------------------------------------------ Line3D::Impl
struct Line3D::Impl {
    l3d_ctx* ctx = nullptr;                               // the primary: ctxs[0]
    std::vector<l3d_ctx*> ctxs; std::vector<int> devices; // one context per listed device (matchImages splits the pairs over them)
    std::string output_folder, err;
    bool load_segments, by_wps, use_gpu, verbose = false;
    int max_img_width; unsigned int max_line_segments;
    std::mutex mtx;                                       // addImage is thread-safe like line3D.cc:129-226
    std::map<unsigned int, HostView> views;               // ascending camID == processing order (line3D.cc:704)
    std::vector<float> views_avg_depths;
    std::map<unsigned int, std::list<unsigned int> > wps2views;
    std::map<unsigned int, std::set<unsigned int> > visual_neighbors;
    // parameters (matchImages / reconstruct3Dlines)
    unsigned int num_neighbors = 10, visibility_t = 3;
    float sigma_p = 2.5f, sigma_a = 10.f, two_sigA_sqr = 200.f, epi = 0.25f, const_reg_depth = -1.f, med_scene_depth = -1.f,
          med_scene_depth_lines = 0.f, collin_t = -1.f;
    bool use_ceres = false;
    int kNN = 10;
    bool fixed3Dreg = false, perform_RDD = false, matched = false;
    Vector3d translation;
    int shard_rank = 0, shard_world = 1; Line3D::MatchExchangeFn exchange = nullptr; void* exchange_user = nullptr;
    // addImage with an image: the detector, the camera IDs whose image is being prepared, and the lock of the GPU step on ctx
    Line3D::SegmentDetectorFn detector = nullptr; void* detector_user = nullptr;
    std::set<unsigned int> reserved;
    std::mutex prep_mtx;
    // addImage with a lens: the source, undistorted and prepared image on the primary device (grow-only, used under prep_mtx)
    struct DeviceScratch {
        void* p = nullptr; size_t cap = 0; int device = 0;
        ~DeviceScratch() { if (p) { int d = 0; cudaGetDevice(&d); cudaSetDevice(device); cudaFree(p); cudaSetDevice(d); } }
    } prep_scratch;
    struct { l3dpp_detect_fn fn; void* user; } c_detector{nullptr, nullptr};   // l3dpp_set_segment_detector
    // setLineCandidates: per view pair (smaller camID, larger camID) its correspondences (segment of the smaller, of the larger); and for
    // the pairs of one matchImages (stage_candidates) the flags, (pair, src_seg, tgt_seg) triples and listed counts of l3d_match_pairs_cand
    std::map<std::pair<unsigned int, unsigned int>, std::vector<std::pair<unsigned int, unsigned int> > > cand_lists;
    std::vector<int32_t> cand_restricted, cand_trip;
    std::vector<long long> cand_count;
    // index maps (rebuilt at matchImages)
    std::vector<HostView*> vlist;                         // by view index (ascending camID)
    std::map<unsigned int, int> index_of;
    std::vector<int32_t> pairs; std::vector<float> F; std::vector<double> F_d;   // (src idx, tgt idx) in match order, 9 entries of F per pair
    // results
    std::vector<l3d_match> est_best; std::vector<double> est_P; std::vector<int> est_index;   // est_index: est_best's entry by global segment, or -1
    Affinity A, A_raw; std::vector<long long> local2global;
    std::vector<FinalLine3D> lines3D;
    Line3DStats st;

    void fail(const std::string& what) { err = what; if (verbose) std::cerr << "[L3D++] ERROR: " << what << std::endl; }
    bool reject(unsigned int camID, const std::string& what) { fail("addImage [" + std::to_string(camID) + "]: " + what); return false; }
    bool chk(long long rc, const char* what) { if (rc < 0) { fail(std::string(what) + ": " + l3d_last_error(ctx)); return false; } return true; }
    void log(const std::string& s) { if (verbose) std::cout << "[L3D++] " << s << std::endl; }

    void shift_all(const Vector3d& d)                     // performTranslation line3D.cc:548-575
    {
        for (auto& kv : views) kv.second.shift(d);
        for (FinalLine3D& L : lines3D) {
            for (Segment3D& s : L.collinear3Dsegments_) s.translate(d);
            L.underlyingCluster_.translate(d);
        }
    }
    struct Translated {                                   // translate (line3D.cc:500-536) for one scope, untranslate (539-545) at its end:
        Impl& P;                                          // the 3D lines made meanwhile move back with the views
        explicit Translated(Impl& p) : P(p)
        {
            if (P.views.empty()) return;
            double tr[3] = {0, 0, 0};
            for (int a = 0; a < 3; ++a) {
                std::vector<double> c;
                for (auto& kv : P.views) { const double v = a == 0 ? kv.second.C.x : (a == 1 ? kv.second.C.y : kv.second.C.z); if (std::fabs(v) > EPS) c.push_back(v); }
                tr[a] = median_of(c, 0.0);
            }
            P.translation = Vector3d(tr[0], tr[1], tr[2]);
            P.shift_all(P.translation * -1.0);
        }
        ~Translated() { P.shift_all(P.translation); }
    };

    float spatial_reg(const HostView& v, float r) const   // View::getSpecificSpatialReg view.cc:307-314
    {
        const Vector3d a = v.ray(v.pp.x, v.pp.y), b = v.ray(v.pp.x + r, v.pp.y);
        return (float)std::sin(std::acos(std::fmin(std::fmax(dot(a, b), -1.0), 1.0)));
    }
    void find_visual_neighbors(unsigned int camID);
    Matrix3d fundamental(const HostView& s, const HostView& t) const   // getFundamentalMatrix line3D.cc:874-892
    {
        const Matrix3d R = matmul(t.R, transposed(s.R));
        const Vector3d tt = t.t - matvec(R, s.t);
        Matrix3d T; T(0, 0) = 0; T(0, 1) = -tt.z; T(0, 2) = tt.y; T(1, 0) = tt.z; T(1, 1) = 0; T(1, 2) = -tt.x; T(2, 0) = -tt.y; T(2, 1) = tt.x; T(2, 2) = 0;
        return matmul(matmul(inverted(transposed(t.K)), matmul(T, R)), inverted(s.K));
    }
    std::vector<l3d_view_desc> descs(std::vector<const float*>* segp = nullptr) const   // segp: each view's segments, for l3d_set_views
    {
        std::vector<l3d_view_desc> d(vlist.size());
        for (size_t i = 0; i < vlist.size(); ++i) {
            const HostView& v = *vlist[i];
            if (segp) segp->push_back(&v.lines[0].v[0]);
            d[i].cam_id = v.id; d[i].width = v.width; d[i].height = v.height; d[i].nseg = (int32_t)v.lines.size();
            memcpy(d[i].RtKinv, v.RtKinv_f, sizeof(v.RtKinv_f)); memcpy(d[i].C, v.C_f3, sizeof(v.C_f3));
            memcpy(d[i].RtKinv_d, v.RtKinv.m, sizeof(v.RtKinv.m));
            d[i].C_d[0] = v.C.x; d[i].C_d[1] = v.C.y; d[i].C_d[2] = v.C.z;
            d[i].k = v.k; d[i].median_depth = v.median_depth;
        }
        return d;
    }
    Segment2D seg_of(long long g) const
    {
        auto it = std::upper_bound(vlist.begin(), vlist.end(), g, [](long long x, const HostView* v) { return x < v->seg_off; });
        const HostView* v = *(it - 1);
        return Segment2D(v->id, (unsigned int)(g - v->seg_off));
    }
    const Segment3D estimate(const Segment2D& s) const
    {
        const int e = est_index[vlist[index_of.at(s.camID())]->seg_off + s.segID()];
        assert(e >= 0);                                   // cluster members come from the affinity matrix: all have an estimate
        return Segment3D(Vector3d(est_P[6 * e], est_P[6 * e + 1], est_P[6 * e + 2]), Vector3d(est_P[6 * e + 3], est_P[6 * e + 4], est_P[6 * e + 5]));
    }
    bool segments_from_image(unsigned int camID, const Image8u& image, const LensDistortion* lens, const Matrix3d& K, Line3D::SegmentDetectorFn fn,
                             void* user, std::vector<Vec4f>& segs, std::string& why);
    bool prepare_undistorted(const Image8u& image, const LensDistortion& lens, const Matrix3d& K, Image8u& gray, std::string& why);
    bool check_lens(unsigned int camID, const LensDistortion& lens, const Matrix3d& K);
    bool line_from_cluster(const std::list<Segment2D>& cluster, LineCluster3D& out) const;
    Segment3D project_onto_line(const Segment2D& s2, const Segment3D& s3, bool& ok) const;
    std::list<Segment3D> collinear_segments(const LineCluster3D& cl) const;
    // addImage's checks under mtx.  Image overload (no_segments null): size, camera ID in views or reservations, world points (line3D.cc:116-155).
    // Segments overload: size, world points, segments (no_segments: why none), then the ID in views only (the image overload calls it reserved).
    bool check_view(unsigned int camID, int w, int h, const std::list<unsigned int>& wps_or_neighbors, const std::string* no_segments)
    {
        const bool in_use = views.count(camID) || (!no_segments && reserved.count(camID));
        const bool rest_ok = !wps_or_neighbors.empty() && (!no_segments || no_segments->empty());
        if (std::max(w, h) < 800) return reject(camID, "image is too small for reliable results (larger side should be >= 800px)");
        if (in_use && (!no_segments || rest_ok)) return reject(camID, "camera ID already in use");
        if (wps_or_neighbors.empty()) return reject(camID, by_wps ? "view has no worldpoints" : "view has no visual neighbors");
        return rest_ok || reject(camID, *no_segments);
    }
    // the view's segment cache, used as stored (detectLineSegments line3D.cc:295-309): true if it was read, with `why` set if the view
    // cannot use what it holds; false with `why` saying why it was not read.  Reads only what is fixed at construction: needs no lock.
    bool read_segment_cache(unsigned int camID, int w, int h, std::vector<Vec4f>& segs, std::string& why) const
    {
        const std::string path = segmentCachePath(output_folder, camID, w, h, max_img_width);
        if (!load_segments) { why = "no line segments given, and load_segments is off so the segment cache " + path + " was not read"; return false; }
        if (!std::ifstream(path.c_str(), std::ios::binary)) { why = "no line segments given and no segment cache " + path + " (line detection is outside this library)"; return false; }
        std::string e;
        if (!readSegmentCache(path, segs, &e)) why = "unreadable segment cache " + e;
        else if (segs.empty()) why = "the segment cache " + path + " holds no segments";
        return true;
    }
    void index_views()                                    // vlist, index_of and every view's global index of its segment 0
    {
        vlist.clear(); index_of.clear();
        long long off = 0;
        for (auto& kv : views) {
            HostView& v = kv.second;
            v.seg_off = off; off += (long long)v.lines.size();
            index_of[v.id] = (int)vlist.size(); vlist.push_back(&v);
        }
    }
    // the view pairs in the reference's order (computeMatches line3D.cc:704-741), F in float and double (861-897, 2775-2781)
    void list_pairs()
    {
        pairs.clear(); F.clear(); F_d.clear();
        std::set<std::pair<unsigned int, unsigned int> > done;
        for (auto& kv : visual_neighbors)
            for (unsigned int n : kv.second) {
                const unsigned int s = kv.first;
                if (n == s || !done.insert(std::make_pair(std::min(s, n), std::max(s, n))).second) continue;
                pairs.push_back(index_of[s]); pairs.push_back(index_of[n]);
                const Matrix3d Fd = fundamental(views[s], views[n]);
                for (int i = 0; i < 9; ++i) { F.push_back((float)Fd.m[i]); F_d.push_back(Fd.m[i]); }
            }
    }
    // The setLineCandidates lists of the pairs of this matchImages as l3d_match_pairs_cand takes them, in the direction list_pairs() chose;
    // false (lastError set) for a segment ID beyond its view's segments.  Lists of pairs not matched are ignored.
    bool stage_candidates()
    {
        cand_restricted.clear(); cand_trip.clear(); cand_count.clear();
        if (cand_lists.empty()) return true;
        const int npairs = (int)(pairs.size() / 2);
        std::map<std::pair<unsigned int, unsigned int>, int> pair_of;
        for (int i = 0; i < npairs; ++i) {
            const unsigned int s = vlist[pairs[2 * i]]->id, t = vlist[pairs[2 * i + 1]]->id;
            pair_of[std::make_pair(std::min(s, t), std::max(s, t))] = i;
        }
        cand_restricted.assign((size_t)npairs, 0); cand_count.assign((size_t)npairs, 0);
        size_t ignored = 0;
        for (const auto& kv : cand_lists) {
            const auto it = pair_of.find(kv.first);
            if (it == pair_of.end()) { ++ignored; continue; }
            const int i = it->second;
            const HostView &vs = *vlist[pairs[2 * i]], &vt = *vlist[pairs[2 * i + 1]];
            const bool fwd = vs.id == kv.first.first;
            cand_restricted[i] = 1; cand_count[i] = (long long)kv.second.size();
            for (const auto& c : kv.second) {
                const unsigned int a = fwd ? c.first : c.second, b = fwd ? c.second : c.first;
                for (const auto& vs_seg : {std::make_pair(&vs, a), std::make_pair(&vt, b)})
                    if (vs_seg.second >= vs_seg.first->lines.size()) {
                        fail("setLineCandidates: segment " + std::to_string(vs_seg.second) + " of camera " + std::to_string(vs_seg.first->id) +
                             " is beyond its " + std::to_string(vs_seg.first->lines.size()) + " segments");
                        return false;
                    }
                cand_trip.push_back(i); cand_trip.push_back((int32_t)a); cand_trip.push_back((int32_t)b);
            }
        }
        if (ignored) log("setLineCandidates: " + std::to_string(ignored) + " candidate list(s) ignored: their view pairs are not matched");
        return true;
    }
    // the pairs [first, last) in `parts` contiguous shares balanced by their cost, Ns*Nt or a restricted pair's listed correspondences:
    // share p is [bounds[p], bounds[p + 1])
    bool split_pairs(int first, int last, int parts, std::vector<int32_t>& bounds)
    {
        std::vector<long long> cost((size_t)(last - first));
        for (int i = first; i < last; ++i)
            cost[i - first] = !cand_restricted.empty() && cand_restricted[i] ? cand_count[i]
                                                                             : (long long)vlist[pairs[2 * i]]->lines.size() * (long long)vlist[pairs[2 * i + 1]]->lines.size();
        bounds.resize((size_t)parts + 1);
        if (!chk(l3d_balanced_split(cost.data(), last - first, parts, bounds.data()), "l3d_balanced_split")) return false;
        for (int32_t& b : bounds) b += first;
        return true;
    }
    // the upload, this rank's share of the pairs (all without setShard) matched on this Line3D's devices, the exchange with the others
    bool match(const std::vector<l3d_view_desc>& d, const std::vector<const float*>& segp, float& ms_gather)
    {
        if (!chk(l3d_set_views(ctx, (int)d.size(), d.data(), segp.data()), "l3d_set_views") || !stage_candidates()) return false;
        const int npairs = (int)(pairs.size() / 2);
        if (shard_world == 1) return match_on_devices(0, npairs, d, segp, ms_gather) && chk(l3d_sync(ctx), "l3d_sync");
        std::vector<int32_t> bounds;
        return split_pairs(0, npairs, shard_world, bounds) && match_on_devices(bounds[shard_rank], bounds[shard_rank + 1], d, segp, ms_gather) &&
               chk(l3d_sync(ctx), "l3d_sync") && exchange_matches(bounds);
    }
    // The pairs [first, last) on the primary, or every device's share (split_pairs) uploaded and matched from its own host thread (keep-all
    // waits on the host between its count and store passes, so one thread would serialise the devices), then gathered on the primary's
    // stream.  The threads share no mutable host state: each works on its own context and writes only its own error slot.
    bool match_on_devices(int first, int last, const std::vector<l3d_view_desc>& d, const std::vector<const float*>& segp, float& ms_gather)
    {
        // use_GPU selects the reference's semantics, not the processor (line3D.cc:708-757): true = K_match_lines / K_score_matches
        // float arithmetic, false = matchingCPU / scoringCPU double arithmetic.  Both run on the GPU.
        const bool cand = !cand_restricted.empty();
        const char* match_what = cand ? (use_gpu ? "l3d_match_pairs_cand" : "l3d_match_pairs_cand_f64") : use_gpu ? "l3d_match_pairs_range" : "l3d_match_pairs_f64";
        const int npairs = (int)(pairs.size() / 2);
        const l3d_match_cand_desc cd = {cand_restricted.data(), cand_trip.data(), (long long)(cand_trip.size() / 3), 0};
        auto match_on = [&](l3d_ctx* c, int f, int l) {
            if (cand)
                return use_gpu ? l3d_match_pairs_cand(c, npairs, pairs.data(), F.data(), epi, kNN, f, l, &cd)
                               : l3d_match_pairs_cand_f64(c, npairs, pairs.data(), F_d.data(), epi, kNN, f, l, &cd);
            return use_gpu ? l3d_match_pairs_range(c, npairs, pairs.data(), F.data(), epi, kNN, f, l)
                           : l3d_match_pairs_f64(c, npairs, pairs.data(), F_d.data(), epi, kNN, f, l);
        };
        if (ctxs.size() == 1) return chk(match_on(ctx, first, last), match_what);
        const int nd = (int)ctxs.size();
        std::vector<int32_t> b;
        if (!split_pairs(first, last, nd, b)) return false;
        std::vector<std::string> errs((size_t)nd);
        auto run = [&](int i) {
            l3d_ctx* c = ctxs[i];
            const char* what = "l3d_set_views";
            long long rc = i == 0 ? 0 : l3d_set_views(c, (int)d.size(), d.data(), segp.data());     // the primary has its views already
            if (rc >= 0) { what = match_what; rc = match_on(c, b[i], b[i + 1]); }
            if (rc >= 0) { what = "l3d_sync"; rc = l3d_sync(c); }
            if (rc < 0) errs[i] = "device " + std::to_string(devices[i]) + " (#" + std::to_string(i) + "): " + what + ": " + l3d_last_error(c);
        };
        std::vector<std::thread> th;
        for (int i = 1; i < nd; ++i) th.emplace_back(run, i);
        run(0);
        for (std::thread& x : th) x.join();
        for (const std::string& e : errs)
            if (!e.empty()) { fail(e); return false; }
        cudaSetDevice(devices[0]);
        cudaStream_t s = (cudaStream_t)l3d_stream(ctx);
        cudaEvent_t e0 = nullptr, e1 = nullptr;
        const bool timed = cudaEventCreate(&e0) == cudaSuccess && cudaEventCreate(&e1) == cudaSuccess && cudaEventRecord(e0, s) == cudaSuccess;
        bool ok = chk(l3d_match_gather(ctx, nd, ctxs.data(), b.data()), "l3d_match_gather");
        cudaSetDevice(devices[0]);
        ok = ok && (!timed || cudaEventRecord(e1, s) == cudaSuccess) && chk(l3d_sync(ctx), "l3d_sync");
        if (ok && timed) cudaEventElapsedTime(&ms_gather, e0, e1);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
        return ok;
    }
    bool exchange_matches(const std::vector<int32_t>& bounds)   // every rank's rows of the match buffers to every rank; bounds: the ranks' shares
    {
        std::vector<long long> row_off(pairs.size() / 2 + 1), row_bounds((size_t)shard_world + 1);
        void *dc = nullptr, *dr = nullptr;
        if (!chk(l3d_pair_row_offsets(ctx, row_off.data()), "l3d_pair_row_offsets") || !chk(l3d_match_device_buffers(ctx, &dc, &dr), "l3d_match_device_buffers")) return false;
        for (int r = 0; r <= shard_world; ++r) row_bounds[r] = row_off[bounds[r]];
        auto send = [&](int knn, const char* what) {
            if (exchange(exchange_user, dc, dr, row_bounds.data(), shard_world, knn) == 0) return true;
            fail(std::string("matchImages: the match exchange callback failed") + what);
            return false;
        };
        if (kNN >= 1 && kNN <= 32) return send(kNN, "");
        // Keep-all and kNN > 32: every rank laid out its records at the longest row of its own share.  Once the counts are exchanged,
        // every rank reduces the same counts to the same stride and re-lays its rows at it; then the records move.
        int stride = 0;
        return send(0, " (row counts)") && chk(stride = l3d_match_restride(ctx, 0), "l3d_match_restride") &&
               chk(l3d_match_device_buffers(ctx, &dc, &dr), "l3d_match_device_buffers") && send(stride, " (records)");
    }
    // every segment's best estimate, then filterMatches' tail (line3D.cc:1657-1668): every view's median depth of them
    bool download_estimates()
    {
        const long long ne = l3d_get_estimates(ctx, nullptr, nullptr, 0);
        if (!chk(ne, "l3d_get_estimates")) return false;
        est_best.resize(ne); est_P.resize(6 * (size_t)ne);
        if (ne && !chk(l3d_get_estimates(ctx, est_best.data(), est_P.data(), ne), "l3d_get_estimates")) return false;
        std::map<unsigned int, std::vector<float> > depths;
        est_index.assign((size_t)(vlist.back()->seg_off + (long long)vlist.back()->lines.size()), -1);
        for (size_t e = 0; e < est_best.size(); ++e) {
            const l3d_match& m = est_best[e];
            depths[m.src_cam].push_back(m.d_p1); depths[m.src_cam].push_back(m.d_p2);
            est_index[views[m.src_cam].seg_off + m.src_seg] = (int)e;
        }
        for (auto& kv : views) {
            kv.second.median_depth = median_of(depths[kv.first], (float)EPS);          // update_median_depth view.h:108-121
            if (fixed3Dreg) kv.second.k = sigma_p / med_scene_depth;
        }
        return true;
    }
    // findCollinearSegments and computingAffinityMatrix (line3D.cc:1751-1756, 1827-1979) on the device; collin_t <= eps: no collinearity
    bool affinity_matrix(const std::vector<l3d_view_desc>& d)
    {
        bool ok = chk(l3d_update_view_params(ctx, (int)d.size(), d.data()), "l3d_update_view_params") &&
                  chk(l3d_find_collinear(ctx, collin_t > EPS ? collin_t : 0.0f, use_gpu ? L3D_SEM_REF_GPU : L3D_SEM_REF_CPU), "l3d_find_collinear");
        st.collinear_entries = ok ? l3d_collinear_total(ctx) : 0;
        long long nids = 0;
        const long long nA = ok ? l3d_affinity_matrix(ctx, two_sigA_sqr, med_scene_depth_lines, MIN_AFFINITY, nullptr, nullptr, nullptr, 0, nullptr, 0, &nids) : -1;
        ok = ok && chk(nA, "l3d_affinity_matrix");
        A = Affinity(); local2global.clear();
        if (ok && nA > 0) {
            A.i.resize((size_t)nA); A.j.resize((size_t)nA); A.w.resize((size_t)nA); local2global.resize((size_t)nids);
            ok = chk(l3d_affinity_matrix(ctx, two_sigA_sqr, med_scene_depth_lines, MIN_AFFINITY, A.i.data(), A.j.data(), A.w.data(), nA,
                                         local2global.data(), nids, &nids), "l3d_affinity_matrix");
        }
        if (!ok) return false;
        A_raw = A;
        st.affinity_entries = (long long)A.w.size(); st.affinity_rows = (long long)local2global.size();
        return true;
    }
    // performRDD (line3D.cc:2026-2076) on the device; one download in the (i, j) order the reference's std::map rebuilds A_ in (2039-2071)
    bool diffuse()
    {
        Affinity D{std::vector<int>(A.w.size()), std::vector<int>(A.w.size()), std::vector<float>(A.w.size())};
        if (!chk(l3d_rdd_affinity(ctx, RDD_MAX_ITER, D.i.data(), D.j.data(), D.w.data(), (long long)D.w.size()), "l3d_rdd_affinity")) return false;
        A = std::move(D);
        return true;
    }
    bool cluster_segments(std::vector<LineCluster3D>& clusters)   // clusterSegments line3D.cc:2079-2152
    {
        st.clusters_total = 0;
        const int n = (int)local2global.size();           // 0 without edges: then there is nothing to cluster
        std::vector<unsigned int> worder;
        if (A.w.size() > (1u << 20)) {          // big list: sort the weights on the device (stable, like std::list::sort)
            worder.resize(A.w.size());
            if (!chk(l3d_argsort_f32(ctx, (long long)A.w.size(), A.w.data(), worder.data()), "l3d_argsort_f32")) return false;
        }
        const std::vector<int> label = segment_graph(A, n, 3.0f, worder.empty() ? nullptr : &worder);
        std::map<int, std::list<Segment2D> > members; std::map<int, std::set<unsigned int> > cams; std::vector<int> order;
        for (int id = 0; id < n; ++id) {
            const int cl = label[id];
            if (!members.count(cl)) order.push_back(cl);
            const Segment2D s = seg_of(local2global[id]);
            members[cl].push_back(s); cams[cl].insert(s.camID());
        }
        st.clusters_total = (long long)order.size();
        std::vector<const std::list<Segment2D>*> todo;
        for (int cl : order) if (cams[cl].size() >= visibility_t) todo.push_back(&members[cl]);
        std::vector<LineCluster3D> fitted(todo.size()); std::vector<unsigned char> good(todo.size(), 0);
        parallel_for(todo.size(), [&](size_t i) { good[i] = line_from_cluster(*todo[i], fitted[i]) ? 1 : 0; });
        for (size_t i = 0; i < todo.size(); ++i) if (good[i]) clusters.push_back(fitted[i]);
        st.clusters_valid = (long long)clusters.size();
        return true;
    }
    // optimizeClusters (line3D.cc:1800-1805, 2269-2275): bundle the cluster lines against their 2D residuals and drop the invalid ones.
    // The reference needs Ceres for this (optimization.cc); here the same problem is minimised on the GPU (l3d_optimize_lines).
    bool optimize_clusters(std::vector<LineCluster3D>& clusters, bool use_CERES, unsigned int max_iter)
    {
        st.opt_iterations = 0; st.opt_cost_before = st.opt_cost_after = 0.0;
        if (!use_CERES || clusters.empty()) return true;
        const int Lc = (int)clusters.size(), nc = (int)vlist.size();
        std::vector<double> p((size_t)6 * Lc), cams((size_t)16 * nc), xy;
        std::vector<long long> ptr((size_t)Lc + 1, 0);
        std::vector<int> rcam;
        for (int v = 0; v < nc; ++v) {
            const HostView& hv = *vlist[v];
            double* cm = &cams[(size_t)16 * v];
            for (int r = 0; r < 3; ++r) for (int c2 = 0; c2 < 3; ++c2) cm[3 * r + c2] = hv.R(r, c2);
            cm[9] = hv.C.x; cm[10] = hv.C.y; cm[11] = hv.C.z;
            cm[12] = hv.K(0, 0); cm[13] = hv.K(1, 1); cm[14] = hv.K(0, 2); cm[15] = hv.K(1, 2);
        }
        for (int i = 0; i < Lc; ++i) {
            const Segment3D s3 = clusters[i].seg3D();
            p[6 * i] = s3.P1().x; p[6 * i + 1] = s3.P1().y; p[6 * i + 2] = s3.P1().z; p[6 * i + 3] = s3.P2().x; p[6 * i + 4] = s3.P2().y; p[6 * i + 5] = s3.P2().z;
            for (const Segment2D& s2 : *clusters[i].residuals()) {
                const int vi = index_of.at(s2.camID());
                const Vec4f& ln = vlist[vi]->lines[s2.segID()];
                rcam.push_back(vi);
                for (int k = 0; k < 4; ++k) xy.push_back((double)ln.v[k]);
            }
            ptr[i + 1] = (long long)rcam.size();
        }
        std::vector<int> valid((size_t)Lc);
        double summ[8];
        if (!chk(l3d_optimize_lines(ctx, Lc, p.data(), ptr.data(), rcam.data(), xy.data(), nc, cams.data(), (int)max_iter, p.data(), valid.data(), summ),
                 "l3d_optimize_lines")) return false;
        std::vector<LineCluster3D> kept;
        for (int i = 0; i < Lc; ++i) {
            if (!valid[i]) continue;                        // optimization.cc:293-298
            clusters[i].update3Dline(Segment3D(Vector3d(p[6 * i], p[6 * i + 1], p[6 * i + 2]), Vector3d(p[6 * i + 3], p[6 * i + 4], p[6 * i + 5])));
            kept.push_back(clusters[i]);
        }
        clusters.swap(kept);
        st.opt_iterations = (long long)summ[0]; st.opt_cost_before = summ[1]; st.opt_cost_after = summ[2];
        return true;
    }
    void final_segments(const std::vector<LineCluster3D>& clusters)   // computeFinal3Dsegments + filterTinySegments (line3D.cc:2278-2339)
    {
        std::vector<std::list<Segment3D> > kept_segs(clusters.size());
        parallel_for(clusters.size(), [&](size_t i) {
            const LineCluster3D& cl = clusters[i];
            std::list<Segment3D> col = collinear_segments(cl);
            if (col.empty()) return;
            const HostView& rv = *vlist[index_of.at(cl.reference_view())];
            for (const Segment3D& s : col) {
                double u1, v1, u2, v2; rv.project(s.P1(), u1, v1); rv.project(s.P2(), u2, v2);
                if (std::sqrt((u1 - u2) * (u1 - u2) + (v1 - v2) * (v1 - v2)) > rv.min_line_length) kept_segs[i].push_back(s);  // projectedLongEnough view.cc:423-428
            }
        });
        for (size_t i = 0; i < clusters.size(); ++i) {
            if (kept_segs[i].empty()) continue;
            FinalLine3D f; f.collinear3Dsegments_ = kept_segs[i]; f.underlyingCluster_ = clusters[i];
            lines3D.push_back(f);
        }
    }
};

// The candidate half of findVisualNeighborsFromWPs (line3D.cc:618-697), shared by the world-point path below and l3d_pose_neighbors
// (pose_select_neighbors): `ranked` holds view v's candidates with more than 4 common points as (camID, score), by score descending with
// ties in ascending camID (the stable sort of line3D.cc:638 over the camID-ordered map); view_of(camID) gives a candidate's HostView.
// The axis gate keeps that order, so it may come after the sort.
template <class ViewOf>
static void select_visual_neighbors(const HostView& v, const std::vector<std::pair<unsigned int, float> >& ranked, unsigned int num_neighbors,
                                    ViewOf view_of, std::set<unsigned int>& out)
{
    struct Cand { unsigned int cam; float score, axis, dist; };
    std::vector<Cand> cand;
    for (const auto& r : ranked) {
        const HostView& o = view_of(r.first);
        Cand c; c.cam = r.first; c.score = r.second;
        c.axis = (float)std::acos(std::fmin(std::fmax(dot(v.ray(v.pp.x, v.pp.y), o.ray(o.pp.x, o.pp.y)), -1.0), 1.0));      // opticalAxesAngle view.cc:457-463
        const Vector3d ct = matvec(v.R, o.C) + v.t;                                                                        // distanceVisualNeighborScore view.cc:487-501
        c.dist = std::fabs((float)ct.x) + std::fabs((float)ct.y);
        if (c.axis < 1.571f) cand.push_back(c);
    }
    if (cand.size() > num_neighbors) {
        const std::vector<Cand> all = cand;
        const float score_t = 0.80f * cand.front().score;
        size_t nbig = 0;
        while (nbig < cand.size() && cand[nbig].score > score_t) ++nbig;
        cand.resize(nbig);
        std::stable_sort(cand.begin(), cand.end(), [](const Cand& a, const Cand& b) { return a.dist > b.dist; });
        if (cand.size() > num_neighbors / 2) cand.resize(num_neighbors / 2);
        cand.insert(cand.end(), all.begin(), all.end());
    }
    const float min_baseline = 0.1f;
    auto baseline = [&](unsigned int b) { return (float)norm(v.C - view_of(b).C); };
    for (size_t i = 0; i < cand.size() && out.size() < num_neighbors; ++i) {
        const unsigned int n = cand[i].cam;
        if (out.count(n) || !(baseline(n) > min_baseline)) continue;
        bool valid = true;
        for (unsigned int u : out) if (!(baseline(u) > min_baseline)) { valid = false; break; }
        if (valid) out.insert(n);
    }
}

// visual neighbours (line3D.cc:463-485): the given ones that were added, or findVisualNeighborsFromWPs (578-699)
void Line3D::Impl::find_visual_neighbors(unsigned int camID)
{
    std::set<unsigned int>& out = visual_neighbors[camID];
    HostView& v = views[camID];
    if (!by_wps) {
        if (out.empty()) for (unsigned int n : v.wps_or_neighbors) if (views.count(n)) out.insert(n);
        return;
    }
    out.clear();
    std::map<unsigned int, unsigned int> common;
    for (unsigned int wp : v.wps_or_neighbors)
        for (unsigned int other : wps2views[wp]) if (other != camID) ++common[other];
    if (common.empty()) return;
    std::vector<std::pair<unsigned int, float> > ranked;
    for (auto& kv : common)
        if (kv.second > 4) ranked.emplace_back(kv.first, 2.0f * float(kv.second) / float(v.wps_or_neighbors.size() + views[kv.first].wps_or_neighbors.size()));
    std::stable_sort(ranked.begin(), ranked.end(), [](const std::pair<unsigned int, float>& a, const std::pair<unsigned int, float>& b) { return a.second > b.second; });
    select_visual_neighbors(v, ranked, num_neighbors, [&](unsigned int cam) -> const HostView& { return views.find(cam)->second; }, out);
}

// K, R, t of a view and what View::View derives from them (view.cc:6-42): the principal point, R^T K^-1, the centre and their float copies
static void set_camera(HostView& v, const Matrix3d& K, const Matrix3d& R, const Vector3d& t)
{
    v.K = K; v.R = R; v.t = t;
    v.pp = Vector3d(K(0, 2), K(1, 2), 1.0);
    const Matrix3d Rt = transposed(R);
    v.RtKinv = matmul(Rt, inverted(K));
    v.C = matvec(Rt, t * -1.0);
    v.C_f3[0] = (float)v.C.x; v.C_f3[1] = (float)v.C.y; v.C_f3[2] = (float)v.C.z;
    for (int i = 0; i < 9; ++i) v.RtKinv_f[i] = (float)v.RtKinv.m[i];
}

void pose_select_neighbors(int n, const l3d_pose_view* views, const long long* cand_off, const PoseCandidate* cand, unsigned int num_neighbors,
                           std::vector<std::vector<unsigned int> >& out)
{
    std::vector<HostView> hv((size_t)n);
    std::map<unsigned int, int> index_of;
    for (int i = 0; i < n; ++i) {
        const l3d_pose_view& d = views[i];
        Matrix3d K, R;
        K(0, 0) = d.fx; K(0, 1) = d.skew; K(0, 2) = d.cx; K(1, 0) = 0.0; K(1, 1) = d.fy; K(1, 2) = d.cy; K(2, 0) = 0.0; K(2, 1) = 0.0; K(2, 2) = 1.0;
        memcpy(R.m, d.R, sizeof(R.m));
        hv[i].id = d.cam_id; hv[i].width = d.width; hv[i].height = d.height;
        set_camera(hv[i], K, R, Vector3d(d.t[0], d.t[1], d.t[2]));
        index_of[d.cam_id] = i;
    }
    out.assign((size_t)n, std::vector<unsigned int>());
    parallel_for((size_t)n, [&](size_t i) {
        std::vector<std::pair<unsigned int, float> > ranked;
        for (long long k = cand_off[i]; k < cand_off[i + 1]; ++k) ranked.emplace_back(cand[k].cam, cand[k].score);
        std::set<unsigned int> nb;
        select_visual_neighbors(hv[i], ranked, num_neighbors, [&](unsigned int cam) -> const HostView& { return hv[index_of.find(cam)->second]; }, nb);
        out[i].assign(nb.begin(), nb.end());
    });
}

// ------------------------------------------------------------------------------------------------ Line3D
Line3D::Line3D(const std::string& output_folder, const bool load_segments, const int max_img_width, const unsigned int max_line_segments,
               const bool neighbors_by_worldpoints, const bool use_GPU, const int cuda_device)
    : Line3D(output_folder, load_segments, max_img_width, max_line_segments, neighbors_by_worldpoints, use_GPU, std::vector<int>(1, cuda_device))
{
}
Line3D::Line3D(const std::string& output_folder, const bool load_segments, const int max_img_width, const unsigned int max_line_segments,
               const bool neighbors_by_worldpoints, const bool use_GPU, const std::vector<int>& cuda_devices)
    : p_(nullptr)
{
    if (cuda_devices.empty()) throw std::invalid_argument("L3DPP::Line3D: the device list is empty");
    p_ = new Impl();
    p_->output_folder = output_folder; p_->load_segments = load_segments; p_->max_img_width = max_img_width;
    p_->max_line_segments = max_line_segments; p_->by_wps = neighbors_by_worldpoints; p_->use_gpu = use_GPU;
    memset(&p_->st, 0, sizeof(p_->st));
    for (const int dev : cuda_devices) {
        l3d_ctx* c = nullptr;
        if (l3d_ctx_create(dev, &c) != L3D_OK) {
            for (l3d_ctx* x : p_->ctxs) l3d_ctx_destroy(x);
            delete p_; p_ = nullptr;
            throw std::runtime_error(cuda_devices.size() == 1 ? std::string("L3DPP::Line3D: no usable CUDA device - this build has no CPU path")
                                                              : "L3DPP::Line3D: no usable CUDA device " + std::to_string(dev) + " - this build has no CPU path");
        }
        p_->ctxs.push_back(c);
    }
    p_->ctx = p_->ctxs[0]; p_->devices = cuda_devices;
}
Line3D::~Line3D() { if (p_) { for (l3d_ctx* c : p_->ctxs) l3d_ctx_destroy(c); delete p_; } }
const Line3DStats& Line3D::stats() const { return p_->st; }
const char* Line3D::lastError() const { return p_->err.c_str(); }
void Line3D::setVerbose(bool v) { p_->verbose = v; }
void Line3D::setShard(int rank, int world, MatchExchangeFn fn, void* user)
{
    Impl& P = *p_;
    std::lock_guard<std::mutex> g(P.mtx);
    P.err.clear();
    if (world < 1 || rank < 0 || rank >= world || (world > 1 && !fn)) { P.fail("setShard: need 0 <= rank < world and an exchange function"); return; }
    P.shard_rank = rank; P.shard_world = world; P.exchange = fn; P.exchange_user = user;
}
size_t Line3D::numImages() { std::lock_guard<std::mutex> g(p_->mtx); return p_->views.size(); }

bool Line3D::addImage(const unsigned int camID, const int w, const int h, const Matrix3d& K, const Matrix3d& R, const Vector3d& t,
                      const float median_depth, const std::list<unsigned int>& wps_or_neighbors, const std::vector<Vec4f>& line_segments)
{
    Impl& P = *p_;
    // everything that needs no shared state first (the reference's frontends call addImage from an OpenMP loop) ...
    HostView v;
    v.id = camID; v.width = w; v.height = h; v.lines = line_segments; v.wps_or_neighbors = wps_or_neighbors;
    std::string no_segments;
    if (line_segments.empty()) P.read_segment_cache(camID, w, h, v.lines, no_segments);
    v.min_line_length = std::sqrt(float((unsigned)w * (unsigned)w + (unsigned)h * (unsigned)h)) * 0.005f;                           // view.cc:17-18
    set_camera(v, K, R, t);
    // ... then one critical section for the checks, the insertion and the error string.  A failure is reported through the return
    // value AND stays in lastError() (a later successful addImage does not clear it) until the next non-addImage call.
    std::lock_guard<std::mutex> g(P.mtx);
    if (!P.check_view(camID, w, h, wps_or_neighbors, &no_segments)) return false;
    if (P.by_wps) for (unsigned int wp : wps_or_neighbors) P.wps2views[wp].push_back(camID);
    P.views[camID] = v;
    P.visual_neighbors[camID];
    P.views_avg_depths.push_back((float)std::fmax((double)median_depth, EPS));
    return true;
}

// the post-processing of detectLineSegments (line3D.cc:320-360, commons.h:135-156): detections in the prepared (w_p x h_p) image are
// scaled to the image's (w x h), their float length must exceed 0.005 * the image diagonal, std::priority_queue orders them longest
// first (equal lengths in the heap's order) and at most max_segments are kept
struct SegmentData2D { float p1x_, p1y_, p2x_, p2y_, length_; };
struct SegmentData2D_comparison { bool operator()(const SegmentData2D& a, const SegmentData2D& b) const { return a.length_ < b.length_; } };
static std::vector<Vec4f> filter_detections(const std::vector<Vec4f>& detections, int w, int h, int w_p, int h_p, unsigned int max_segments)
{
    const float upscale_x = float(w) / float(w_p), upscale_y = float(h) / float(h_p);
    const float min_len = sqrtf(float(h * h) + float(w * w)) * 0.005f;                   // L3D_DEF_MIN_LINE_LENGTH_FACTOR
    std::priority_queue<SegmentData2D, std::vector<SegmentData2D>, SegmentData2D_comparison> sorted;
    for (const Vec4f& d : detections) {
        SegmentData2D s;
        s.p1x_ = d.v[0] * upscale_x; s.p1y_ = d.v[1] * upscale_y; s.p2x_ = d.v[2] * upscale_x; s.p2y_ = d.v[3] * upscale_y;
        const float dx = s.p1x_ - s.p2x_, dy = s.p1y_ - s.p2y_;
        s.length_ = sqrtf(dx * dx + dy * dy);
        if (s.length_ > min_len) sorted.push(s);
    }
    std::vector<Vec4f> out;
    out.reserve(std::min<size_t>(sorted.size(), max_segments));
    while (!sorted.empty() && out.size() < max_segments) {
        const SegmentData2D& s = sorted.top();
        out.push_back(Vec4f{{s.p1x_, s.p1y_, s.p2x_, s.p2y_}});
        sorted.pop();
    }
    return out;
}

// the segments of an image without given segments (detectLineSegments line3D.cc:249-372): the segment cache, or the prepared image
// through the detector and the post-processing, then the cache is written.  false with `why` set if the view has to be rejected.
bool Line3D::Impl::segments_from_image(unsigned int camID, const Image8u& image, const LensDistortion* lens, const Matrix3d& K,
                                       Line3D::SegmentDetectorFn fn, void* user, std::vector<Vec4f>& segs, std::string& why)
{
    const int w = image.cols, h = image.rows;
    if (image.channels != 1 && image.channels != 3) {                                                     // line3D.cc:251-266
        why = "image type not supported: " + std::to_string(image.channels) + " channels (8-bit grey or RGB images only)";
        return false;
    }
    if (read_segment_cache(camID, w, h, segs, why)) return why.empty();        // a cache that exists decides, usable or not
    if (!fn) return false;
    if (image.data.size() != (size_t)w * h * image.channels) { why = "the pixel buffer does not match rows x cols x channels"; return false; }
    int w_p, h_p;
    preparedImageSize(w, h, max_img_width, w_p, h_p);
    Image8u gray(h_p, w_p, 1);
    if (lens) {
        if (!prepare_undistorted(image, *lens, K, gray, why)) return false;
    } else {
        // the primary context is single-owner: one preparation at a time
        std::lock_guard<std::mutex> g(prep_mtx);
        l3d_image_prep_desc d;
        std::memset(&d, 0, sizeof(d));
        d.width = w; d.height = h; d.channels = image.channels; d.max_img_width = max_img_width;
        d.src_pitch = (int64_t)w * image.channels; d.dst_pitch = w_p;
        d.src = image.data.data(); d.dst = gray.data.data();
        d.out_width = w_p; d.out_height = h_p;
        if (l3d_prepare_gray_u8(ctx, 1, &d, 0) != L3D_OK) { why = std::string("image preparation: ") + l3d_last_error(ctx); return false; }
    }
    std::vector<Vec4f> detections;
    if (!fn(user, gray, detections)) { why = "the segment detector failed"; return false; }
    segs = filter_detections(detections, w, h, w_p, h_p, max_line_segments);
    if (segs.empty()) {
        why = "none of the " + std::to_string(detections.size()) + " detected segments is longer than 0.005 * the image diagonal";
        return false;
    }
    if (load_segments) {                                                                                  // line3D.cc:363-366
        std::string e;
        mkdir((output_folder + "/L3D++_data").c_str(), 0777);     // the reference's constructor creates it (line3D.cc:59-61)
        if (!writeSegmentCache(segmentCachePath(output_folder, camID, w, h, max_img_width), segs, &e)) log("WARNING: segment cache not written: " + e);
    }
    return true;
}

// the camera, lens and new-K fields of an l3d_undistort_desc (include/l3d_capi.h); the image fields are zero
static l3d_undistort_desc lens_desc(const LensDistortion& lens, const Matrix3d& K, const Matrix3d& newK)
{
    l3d_undistort_desc d;
    std::memset(&d, 0, sizeof(d));
    d.fx = K(0, 0); d.fy = K(1, 1); d.cx = K(0, 2); d.cy = K(1, 2);
    d.new_fx = newK(0, 0); d.new_fy = newK(1, 1); d.new_cx = newK(0, 2); d.new_cy = newK(1, 2);
    d.model = lens.model;
    d.tangential[0] = lens.p[0]; d.tangential[1] = lens.p[1];
    if (lens.model == LensDistortion::FISHEYE) {   // k[4], k[5] go where l3d_undistort_u8 rejects them if nonzero
        for (int k = 0; k < 4; ++k) d.fisheye[k] = lens.k[k];
        d.radial[0] = lens.k[4]; d.radial[1] = lens.k[5];
    } else {
        for (int k = 0; k < 3; ++k) { d.radial[k] = lens.k[k]; d.rational[k] = lens.k[3 + k]; }
    }
    return d;
}

// a zero-initialised LensDistortion: no distortion at all (a fisheye lens with k = 0 still is one)
static bool lens_is_zero(const LensDistortion& lens)
{
    bool zero = lens.model == LensDistortion::RADTAN && lens.p[0] == 0.0 && lens.p[1] == 0.0;
    for (int k = 0; k < 6; ++k) zero = zero && lens.k[k] == 0.0;
    return zero;
}

// the lens of an addImage call, checked as l3d_undistort_u8 checks it (an empty point set: no GPU work); false: the view is rejected
bool Line3D::Impl::check_lens(unsigned int camID, const LensDistortion& lens, const Matrix3d& K)
{
    l3d_points_desc d;
    std::memset(&d, 0, sizeof(d));
    d.cam = lens_desc(lens, K, Matrix3d());
    std::string why;
    {
        std::lock_guard<std::mutex> g(prep_mtx);
        if (l3d_undistort_points(ctx, 1, &d, 0) == L3D_OK) return true;
        why = std::string("lens: ") + l3d_last_error(ctx);
    }
    std::lock_guard<std::mutex> g(mtx);
    return reject(camID, why);
}

// The image undistorted into K and prepared for the detector on the primary device, the undistorted image never leaving it: one upload,
// l3d_undistort_u8 and l3d_prepare_gray_u8 on device buffers, one download of the prepared image into gray (sized by the caller).
bool Line3D::Impl::prepare_undistorted(const Image8u& image, const LensDistortion& lens, const Matrix3d& K, Image8u& gray, std::string& why)
{
    const int w = image.cols, h = image.rows, ch = image.channels;
    const size_t in_bytes = (size_t)w * h * ch, gray_bytes = gray.data.size();
    std::lock_guard<std::mutex> g(prep_mtx);                  // the primary context is single-owner: one preparation at a time
    int prev = 0;
    cudaGetDevice(&prev);
    struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};
    cudaSetDevice(devices[0]);
    DeviceScratch& s = prep_scratch;
    if (s.cap < 2 * in_bytes + gray_bytes) {
        if (s.p) cudaFree(s.p);
        s.p = nullptr; s.cap = 0; s.device = devices[0];
        if (cudaMalloc(&s.p, 2 * in_bytes + gray_bytes) != cudaSuccess) { s.p = nullptr; why = "lens undistortion: out of device memory"; return false; }
        s.cap = 2 * in_bytes + gray_bytes;
    }
    unsigned char* src = (unsigned char*)s.p;
    unsigned char* und = src + in_bytes;
    unsigned char* dst = und + in_bytes;
    cudaStream_t st = (cudaStream_t)l3d_stream(ctx);
    if (cudaMemcpyAsync(src, image.data.data(), in_bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) { why = "lens undistortion: upload failed"; return false; }
    l3d_undistort_desc u = lens_desc(lens, K, Matrix3d());
    u.width = w; u.height = h; u.channels = ch;
    u.src_pitch = u.dst_pitch = (int64_t)w * ch;
    u.src = src; u.dst = und;
    if (l3d_undistort_u8(ctx, 1, &u, 1) != L3D_OK) { why = std::string("lens undistortion: ") + l3d_last_error(ctx); return false; }
    l3d_image_prep_desc d;
    std::memset(&d, 0, sizeof(d));
    d.width = w; d.height = h; d.channels = ch; d.max_img_width = max_img_width;
    d.src_pitch = (int64_t)w * ch; d.dst_pitch = gray.cols;
    d.src = und; d.dst = dst;
    d.out_width = gray.cols; d.out_height = gray.rows;
    if (l3d_prepare_gray_u8(ctx, 1, &d, 1) != L3D_OK) { why = std::string("image preparation: ") + l3d_last_error(ctx); return false; }
    if (cudaMemcpyAsync(gray.data.data(), dst, gray_bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess || l3d_sync(ctx) != L3D_OK) {
        why = "lens undistortion: download failed";
        return false;
    }
    return true;
}

bool Line3D::addImage(const unsigned int camID, const Image8u& image, const Matrix3d& K, const Matrix3d& R, const Vector3d& t,
                      const float median_depth, const std::list<unsigned int>& wps_or_neighbors, const std::vector<Vec4f>& line_segments)
{
    LensDistortion none;
    std::memset(&none, 0, sizeof(none));
    return addImage(camID, image, K, R, t, median_depth, wps_or_neighbors, none, line_segments);
}

bool Line3D::addImage(const unsigned int camID, const int w, const int h, const Matrix3d& K, const Matrix3d& R, const Vector3d& t,
                      const float median_depth, const std::list<unsigned int>& wps_or_neighbors, const LensDistortion& lens,
                      const std::vector<Vec4f>& line_segments)
{
    if (lens_is_zero(lens) || line_segments.empty()) {
        if (!lens_is_zero(lens) && !p_->check_lens(camID, lens, K)) return false;
        return addImage(camID, w, h, K, R, t, median_depth, wps_or_neighbors, line_segments);
    }
    Impl& P = *p_;
    std::vector<Vec4f> segs(line_segments);
    l3d_points_desc d;
    std::memset(&d, 0, sizeof(d));
    d.cam = lens_desc(lens, K, Matrix3d());
    d.count = 2 * (int64_t)segs.size();
    d.src = d.dst = &segs[0].v[0];
    std::string why;
    {
        std::lock_guard<std::mutex> g(P.prep_mtx);
        if (l3d_undistort_points(P.ctx, 1, &d, 0) != L3D_OK) why = std::string("lens: ") + l3d_last_error(P.ctx);
    }
    if (!why.empty()) {
        std::lock_guard<std::mutex> g(P.mtx);
        return P.reject(camID, why);
    }
    return addImage(camID, w, h, K, R, t, median_depth, wps_or_neighbors, segs);
}

bool Line3D::addImage(const unsigned int camID, const Image8u& image, const Matrix3d& K, const Matrix3d& R, const Vector3d& t,
                      const float median_depth, const std::list<unsigned int>& wps_or_neighbors, const LensDistortion& lens,
                      const std::vector<Vec4f>& line_segments)
{
    Impl& P = *p_;
    const int w = image.cols, h = image.rows;
    const bool undistort = !lens_is_zero(lens);
    if (!line_segments.empty()) {
        if (undistort) return addImage(camID, w, h, K, R, t, median_depth, wps_or_neighbors, lens, line_segments);
        return addImage(camID, w, h, K, R, t, median_depth, wps_or_neighbors, line_segments);
    }
    if (undistort && !P.check_lens(camID, lens, K)) return false;
    // the checks before any image work; the camera ID stays reserved until the view is added or rejected
    Line3D::SegmentDetectorFn fn;
    void* user;
    {
        std::lock_guard<std::mutex> g(P.mtx);
        if (!P.check_view(camID, w, h, wps_or_neighbors, nullptr)) return false;
        P.reserved.insert(camID);
        fn = P.detector; user = P.detector_user;
    }
    struct Release {
        Impl& P; unsigned int id;
        ~Release() { std::lock_guard<std::mutex> g(P.mtx); P.reserved.erase(id); }
    } release{P, camID};
    std::vector<Vec4f> segs;
    std::string why;
    if (!P.segments_from_image(camID, image, undistort ? &lens : nullptr, K, fn, user, segs, why)) {
        std::lock_guard<std::mutex> g(P.mtx);
        return P.reject(camID, why);
    }
    return addImage(camID, w, h, K, R, t, median_depth, wps_or_neighbors, segs);
}

void Line3D::setSegmentDetector(SegmentDetectorFn detector, void* user)
{
    Impl& P = *p_;
    std::lock_guard<std::mutex> g(P.mtx);
    P.err.clear();
    P.detector = detector; P.detector_user = user;
}

void Line3D::setLineCandidates(const unsigned int camA, const unsigned int camB, const std::vector<std::pair<unsigned int, unsigned int> >& seg_pairs)
{
    Impl& P = *p_;
    std::lock_guard<std::mutex> g(P.mtx);
    P.err.clear();
    if (camA == camB) { P.fail("setLineCandidates: camA == camB (" + std::to_string(camA) + "): a view pair needs two cameras"); return; }
    std::vector<std::pair<unsigned int, unsigned int> >& L = P.cand_lists[std::make_pair(std::min(camA, camB), std::max(camA, camB))];
    L.clear();
    L.reserve(seg_pairs.size());
    for (const auto& c : seg_pairs) L.push_back(camA < camB ? c : std::make_pair(c.second, c.first));
}

void Line3D::clearLineCandidates()
{
    Impl& P = *p_;
    std::lock_guard<std::mutex> g(P.mtx);
    P.err.clear();
    P.cand_lists.clear();
}

void Line3D::matchImages(const float sigma_position, const float sigma_angle, const unsigned int num_neighbors, const float epipolar_overlap,
                         const int kNN, const float const_regularization_depth)
{
    Impl& P = *p_;
    std::lock_guard<std::mutex> g(P.mtx);
    P.err.clear();
    if (P.views.empty()) { P.fail("no images to match"); return; }
    // parameter checks: line3D.cc:394-413
    P.num_neighbors = (unsigned int)std::max(int(num_neighbors), 2);
    P.sigma_p = sigma_position; P.sigma_a = std::fmin(std::fabs(sigma_angle), 90.0f);
    P.two_sigA_sqr = 2.0f * P.sigma_a * P.sigma_a;
    P.epi = std::fmin(std::fabs(epipolar_overlap), 0.99f); P.kNN = kNN; P.const_reg_depth = const_regularization_depth;
    if (P.sigma_p < 0.0f) { P.fixed3Dreg = true; P.sigma_p = std::fabs(P.sigma_p); } else { P.fixed3Dreg = false; P.sigma_p = std::fmax(0.1f, P.sigma_p); }
    P.med_scene_depth = const_regularization_depth;
    if (const_regularization_depth < 0.0f && P.fixed3Dreg) P.med_scene_depth = median_of(P.views_avg_depths, P.med_scene_depth);
    for (auto& kv : P.views) kv.second.k = P.fixed3Dreg ? P.sigma_p / P.med_scene_depth : P.spatial_reg(kv.second, P.sigma_p);   // view.cc:301-314
    P.matched = false; P.est_best.clear(); P.est_P.clear(); P.est_index.clear();
    const Impl::Translated frame(P);
    P.index_views();
    for (auto& kv : P.views) P.find_visual_neighbors(kv.first);
    P.list_pairs();
    float ms_gather = 0.0f;
    std::vector<const float*> segp;
    const std::vector<l3d_view_desc> d = P.descs(&segp);
    const auto t0 = std::chrono::steady_clock::now();
    nvtxRangePushA("l3d:set_views+match");
    bool ok = P.match(d, segp, ms_gather);
    const auto t1 = std::chrono::steady_clock::now();
    nvtxRangePop(); nvtxRangePushA("l3d:score_sweep");
    ok = ok && P.chk(l3d_score_sweep(P.ctx, P.two_sigA_sqr, MIN_SIMILARITY_3D, MIN_BEST_SCORE_3D, MIN_BEST_SCORE_PERC), "l3d_score_sweep");
    nvtxRangePop();
    const auto t2 = std::chrono::steady_clock::now();
    if (!ok || !P.download_estimates()) return;
    P.st.view_pairs = (long long)(P.pairs.size() / 2); P.st.pair_evaluations = l3d_match_pair_evals(P.ctx); P.st.estimates = (long long)P.est_best.size();
    P.st.matches_after_knn = l3d_match_total_matches(P.ctx);      // reduced on the device (was: download of the whole count array)
    P.st.ms_match = std::chrono::duration<double, std::milli>(t1 - t0).count();
    P.st.ms_score = std::chrono::duration<double, std::milli>(t2 - t1).count();
    P.st.ms_gather = ms_gather;
    P.matched = true;
}

// get3DlineFromCluster (line3D.cc:2155-2218)
bool Line3D::Impl::line_from_cluster(const std::list<Segment2D>& cluster, LineCluster3D& out) const
{
    Vector3d cog(0, 0, 0);
    std::vector<Vector3d> pts;
    unsigned int reference_cam = 0; float max_len_2D = 0.0f;
    for (const Segment2D& s : cluster) {
        const Segment3D h = estimate(s);
        cog = cog + h.P1(); cog = cog + h.P2();
        pts.push_back(h.P1()); pts.push_back(h.P2());
        const Vec4f c = vlist[index_of.at(s.camID())]->lines[s.segID()];
        const float l2 = (c.v[0] - c.v[2]) * (c.v[0] - c.v[2]) + (c.v[1] - c.v[3]) * (c.v[1] - c.v[3]);
        if (l2 > max_len_2D) { max_len_2D = l2; reference_cam = s.camID(); }
    }
    const double n = double(pts.size());
    cog = Vector3d(cog.x / n, cog.y / n, cog.z / n);
    double Sc[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (const Vector3d& p : pts) {
        const double d[3] = {p.x - cog.x, p.y - cog.y, p.z - cog.z};
        for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) Sc[a][b] += d[a] * d[b];
    }
    const Vector3d dir = principal_axis(Sc);
    out = LineCluster3D(Segment3D(cog - dir, cog + dir), cluster, reference_cam);
    return out.size() > 0;
}

// project2DsegmentOnto3Dline (line3D.cc:2221-2266): closest points between the 3D line and the two viewing rays
Segment3D Line3D::Impl::project_onto_line(const Segment2D& s2, const Segment3D& s3, bool& ok) const
{
    const HostView& v = *vlist[index_of.at(s2.camID())];
    const Vec4f l = v.lines[s2.segID()];
    const Vector3d Pl = s3.P1(), u = s3.dir(), w = Pl - v.C;
    const Vector3d v1 = v.ray(l.v[0], l.v[1]), v2 = v.ray(l.v[2], l.v[3]);
    const double a = dot(u, u), b1 = dot(u, v1), b2 = dot(u, v2), c1 = dot(v1, v1), c2 = dot(v2, v2), d = dot(u, w), e1 = dot(v1, w), e2 = dot(v2, w);
    const double den1 = a * c1 - b1 * b1, den2 = a * c2 - b2 * b2;
    ok = std::fabs(den1) > EPS && std::fabs(den2) > EPS;
    if (!ok) return Segment3D();
    return Segment3D(Pl + u * ((b1 * e1 - c1 * d) / den1), Pl + u * ((b2 * e2 - c2 * d) / den2));
}

// findCollinearSegments(cluster) (line3D.cc:2342-2452): sweep along the line, a 3D segment is open while >= 3 cameras see it
std::list<Segment3D> Line3D::Impl::collinear_segments(const LineCluster3D& cl) const
{
    std::list<Segment3D> out;
    const Vector3d cog = (cl.seg3D().P1() + cl.seg3D().P2()) * 0.5;
    struct Pt { size_t line, point, cam; float dist; };
    std::vector<Pt> ev;
    std::vector<Vector3d> pts(cl.residuals()->size() * 2);
    float far = 0.0f; Vector3d border(0, 0, 0);
    size_t id = 0, pid = 0;
    for (const Segment2D& s : *cl.residuals()) {
        bool ok; const Segment3D pr = project_onto_line(s, cl.seg3D(), ok);
        if (ok) {
            const Vector3d e[2] = {pr.P1(), pr.P2()};
            for (int k = 0; k < 2; ++k) {
                pts[pid + k] = e[k];
                Pt p = {id, pid + k, s.camID(), 0.0f}; ev.push_back(p);
                const float dd = (float)norm(e[k] - cog);
                if (dd > far) { far = dd; border = e[k]; }
            }
        }
        ++id; pid += 2;
    }
    if (ev.size() < 6) return out;
    for (Pt& p : ev) p.dist = (float)norm(pts[p.point] - border);
    std::stable_sort(ev.begin(), ev.end(), [](const Pt& a, const Pt& b) { return a.dist < b.dist; });
    std::map<size_t, unsigned int> open_cams; std::set<size_t> open_lines;
    bool opened = false; Vector3d start(0, 0, 0);
    for (const Pt& p : ev) {
        if (!open_lines.count(p.line)) { open_lines.insert(p.line); ++open_cams[p.cam]; }
        else { open_lines.erase(p.line); if (--open_cams[p.cam] == 0) open_cams.erase(p.cam); }
        if (opened && open_cams.size() < 3) { out.push_back(Segment3D(start, pts[p.point])); opened = false; }
        else if (!opened && open_cams.size() >= 3) { start = pts[p.point]; opened = true; }
    }
    return out;
}

void Line3D::reconstruct3Dlines(const unsigned int visibility_t, const bool perform_diffusion, const float collinearity_t, const bool use_CERES,
                                const unsigned int max_iter_CERES)
{
    Impl& P = *p_;
    std::lock_guard<std::mutex> g(P.mtx);
    P.err.clear();
    if (!P.matched || P.est_best.empty()) { P.fail("no clusterable segments! forgot to match lines?"); return; }   // line3D.cc:1712-1718
    P.visibility_t = (unsigned int)std::max(int(visibility_t), 3);
    P.lines3D.clear(); P.collin_t = collinearity_t;
    P.perform_RDD = perform_diffusion && P.use_gpu;                                       // line3D.cc:1729
    const Impl::Translated frame(P);
    std::vector<float> sd;                                // median scene depth for lines (line3D.cc:1759-1774)
    for (auto& kv : P.views) if (kv.second.median_depth > EPS) sd.push_back(kv.second.median_depth);
    P.med_scene_depth_lines = median_of(sd, 0.0f);
    const std::vector<l3d_view_desc> d = P.descs();
    const auto t0 = std::chrono::steady_clock::now();
    if (!P.affinity_matrix(d)) return;
    const auto t1 = std::chrono::steady_clock::now();
    if (P.perform_RDD && !P.A.w.empty() && !P.diffuse()) return;
    const auto t2 = std::chrono::steady_clock::now();
    std::vector<LineCluster3D> clusters;
    if (!P.cluster_segments(clusters) || !P.optimize_clusters(clusters, use_CERES, max_iter_CERES)) return;
    P.use_ceres = use_CERES;
    P.final_segments(clusters);
    const auto t3 = std::chrono::steady_clock::now();
    P.st.lines3D = (long long)P.lines3D.size();
    P.st.ms_affinity = std::chrono::duration<double, std::milli>(t1 - t0).count();
    P.st.ms_diffusion = std::chrono::duration<double, std::milli>(t2 - t1).count();
    P.st.ms_cluster = std::chrono::duration<double, std::milli>(t3 - t2).count();
}

void Line3D::get3Dlines(std::vector<FinalLine3D>& result) { std::lock_guard<std::mutex> g(p_->mtx); result = p_->lines3D; }

Vector4f Line3D::getSegmentCoords2D(const unsigned int camID, const unsigned int segID)
{
    Vector4f c = {{0, 0, 0, 0}};
    auto it = p_->views.find(camID);
    if (it != p_->views.end() && segID < it->second.lines.size()) memcpy(c.v, it->second.lines[segID].v, sizeof(c.v));
    return c;
}
Vector4f Line3D::getSegmentCoords2D(const Segment2D& s) { return getSegmentCoords2D(s.camID(), s.segID()); }

std::string Line3D::createOutputFilename()   // line3D.cc:2855-2894
{
    Impl& P = *p_;
    std::stringstream s;
    s << "Line3D++__";
    if (P.max_img_width > 0) s << "W_" << P.max_img_width << "__"; else s << "W_FULL__";
    s << "N_" << P.num_neighbors << "__" << "sigmaP_" << P.sigma_p << "__" << "sigmaA_" << P.sigma_a << "__" << "epiOverlap_" << P.epi << "__";
    if (P.kNN > 0) s << "kNN_" << P.kNN << "__";
    if (P.collin_t > EPS) s << "COLLIN_" << P.collin_t << "__";
    if (P.use_ceres) s << "OPTIMIZED__";                                   // line3D.cc:2889-2890
    if (P.fixed3Dreg) { s << "FXD_SIGMA_P__"; if (P.const_reg_depth > 0.0f) s << "REG_DEPTH_" << P.const_reg_depth << "__"; }
    if (P.perform_RDD) s << "DIFFUSION__";
    s << "vis_" << P.visibility_t;
    return s.str();
}

void Line3D::save3DLinesAsTXT(const std::string& folder)   // line3D.cc:2631-2687; format README.md:272-277
{
    std::lock_guard<std::mutex> g(p_->mtx);
    p_->err.clear();
    if (p_->lines3D.empty()) { p_->fail("no 3D lines to save!"); return; }
    const std::string path = folder + "/" + createOutputFilename() + ".txt";
    std::ofstream f(path.c_str());
    if (!f) { p_->fail("cannot open " + path + " for writing"); return; }
    for (const FinalLine3D& L : p_->lines3D) {
        if (L.collinear3Dsegments_.empty()) continue;
        f << L.collinear3Dsegments_.size() << " ";
        for (const Segment3D& s : L.collinear3Dsegments_) f << s.P1().x << " " << s.P1().y << " " << s.P1().z << " " << s.P2().x << " " << s.P2().y << " " << s.P2().z << " ";
        f << L.underlyingCluster_.residuals()->size() << " ";
        for (const Segment2D& r : *L.underlyingCluster_.residuals()) {
            const Vector4f c = getSegmentCoords2D(r);
            f << r.camID() << " " << r.segID() << " " << c.v[0] << " " << c.v[1] << " " << c.v[2] << " " << c.v[3] << " ";
        }
        f << std::endl;
    }
}

// the reference's Boost binary archive of lines3D_ (line3D.cc:2690-2711), written by csrc/line3d_bin.cc
void Line3D::save3DLinesAsBIN(const std::string& folder)
{
    std::lock_guard<std::mutex> g(p_->mtx);
    p_->err.clear();
    if (p_->lines3D.empty()) { p_->fail("no 3D lines to save!"); return; }
    std::string e;
    if (!write3DLinesBIN(folder + "/" + createOutputFilename() + ".bin", p_->lines3D, &e)) p_->fail(e);
}

// Wavefront OBJ as the reference writes it (line3D.cc:2568-2628): all vertices first ("v x y z", two per 3D segment,
// default ostream formatting), then one "l a b" element per segment with 1-based vertex indices.
void Line3D::saveResultAsOBJ(const std::string& folder)
{
    std::lock_guard<std::mutex> g(p_->mtx);
    p_->err.clear();
    if (p_->lines3D.empty()) { p_->fail("no 3D lines to save!"); return; }
    const std::string path = folder + "/" + createOutputFilename() + ".obj";
    std::ofstream f(path.c_str());
    if (!f) { p_->fail("cannot open " + path + " for writing"); return; }
    size_t nseg = 0;
    for (const FinalLine3D& L : p_->lines3D)
        for (const Segment3D& s : L.collinear3Dsegments_) {
            const Vector3d e[2] = {s.P1(), s.P2()};
            for (const Vector3d& v : e) f << "v " << v.x << " " << v.y << " " << v.z << std::endl;
            ++nseg;
        }
    for (size_t i = 0; i < nseg; ++i) f << "l " << 2 * i + 1 << " " << 2 * i + 2 << std::endl;
}

// ASCII STL as the reference writes it (line3D.cc:2465-2528): every 3D segment is a degenerate facet P1,P2,P1 with a
// fixed normal, coordinates printed with %e.
void Line3D::saveResultAsSTL(const std::string& folder)
{
    std::lock_guard<std::mutex> g(p_->mtx);
    p_->err.clear();
    if (p_->lines3D.empty()) { p_->fail("no 3D lines to save!"); return; }
    const std::string path = folder + "/" + createOutputFilename() + ".stl";
    std::ofstream f(path.c_str());
    if (!f) { p_->fail("cannot open " + path + " for writing"); return; }
    auto vertex = [&f](const Vector3d& v) { char b[200]; snprintf(b, sizeof(b), "   vertex %e %e %e", v.x, v.y, v.z); f << b << std::endl; };
    f << "solid lineModel" << std::endl;
    for (const FinalLine3D& L : p_->lines3D)
        for (const Segment3D& s : L.collinear3Dsegments_) {
            f << " facet normal 1.0e+000 0.0e+000 0.0e+000" << std::endl << "  outer loop" << std::endl;
            vertex(s.P1()); vertex(s.P2()); vertex(s.P1());
            f << "  endloop" << std::endl << " endfacet" << std::endl;
        }
    f << "endsolid lineModel" << std::endl;
}

void Line3D::undistortImage(const Image8u& in, Image8u& out, const Vector3d& radial, const Vector2d& tangential, const Matrix3d& K)
{
    LensDistortion lens;
    std::memset(&lens, 0, sizeof(lens));
    lens.model = LensDistortion::RADTAN;
    lens.k[0] = radial.x; lens.k[1] = radial.y; lens.k[2] = radial.z; lens.p[0] = tangential.x; lens.p[1] = tangential.y;
    undistortImage(in, out, lens, K);
}

void Line3D::undistortImage(const Image8u& in, Image8u& out, const LensDistortion& lens, const Matrix3d& K)
{
    Matrix3d none;
    std::memset(&none, 0, sizeof(none));
    undistortImage(in, out, lens, K, none, 0, 0);
}

void Line3D::undistortImage(const Image8u& in, Image8u& out, const LensDistortion& lens, const Matrix3d& K, const Matrix3d& newK, int out_width,
                            int out_height)
{
    if (in.data.size() != (size_t)in.rows * in.cols * in.channels || in.rows < 0 || in.cols < 0)
        throw std::invalid_argument("undistortImage: the pixel buffer does not match rows x cols x channels");
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) throw std::runtime_error("undistortImage: no usable CUDA device");
    l3d_ctx* ctx = nullptr;
    if (l3d_ctx_create(dev, &ctx) != L3D_OK) throw std::runtime_error("undistortImage: no usable CUDA device");
    // a separate buffer: in and out may be the same image.  A size l3d_undistort_u8 rejects gets an empty one; the call fails.
    const bool size_ok = (out_width == 0 && out_height == 0) || (out_width >= 1 && out_width <= 32767 && out_height >= 1 && out_height <= 32767);
    const int ow = out_width == 0 && out_height == 0 ? in.cols : out_width, oh = out_width == 0 && out_height == 0 ? in.rows : out_height;
    Image8u res(size_ok ? oh : 0, size_ok ? ow : 0, in.channels);
    l3d_undistort_desc d = lens_desc(lens, K, newK);
    d.width = in.cols; d.height = in.rows; d.channels = in.channels;
    d.src_pitch = (int64_t)in.cols * in.channels;
    d.dst_pitch = (int64_t)(size_ok ? ow : in.cols) * in.channels;
    d.src = in.data.data(); d.dst = res.data.data();
    d.out_width = out_width; d.out_height = out_height;
    const int rc = l3d_undistort_u8(ctx, 1, &d, 0);
    const std::string msg = std::string("undistortImage: ") + l3d_last_error(ctx);
    l3d_ctx_destroy(ctx);
    if (rc == L3D_ERR_INVALID) throw std::invalid_argument(msg);
    if (rc != L3D_OK) throw std::runtime_error(msg);
    out = std::move(res);
}

// l3d_undistort_points of host point sets on the calling thread's device, through a context that lives for the call
static void undistort_point_sets(std::vector<l3d_points_desc>& sets)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) throw std::runtime_error("undistortPoints: no usable CUDA device");
    l3d_ctx* ctx = nullptr;
    if (l3d_ctx_create(dev, &ctx) != L3D_OK) throw std::runtime_error("undistortPoints: no usable CUDA device");
    const int rc = l3d_undistort_points(ctx, (int)sets.size(), sets.data(), 0);
    const std::string msg = std::string("undistortPoints: ") + l3d_last_error(ctx);
    l3d_ctx_destroy(ctx);
    if (rc == L3D_ERR_INVALID) throw std::invalid_argument(msg);
    if (rc != L3D_OK) throw std::runtime_error(msg);
}

void Line3D::undistortPoints(std::vector<float>& xy, const LensDistortion& lens, const Matrix3d& K, const Matrix3d& newK)
{
    if (xy.size() % 2) throw std::invalid_argument("undistortPoints: an odd number of coordinates");
    std::vector<l3d_points_desc> d(1);
    d[0].cam = lens_desc(lens, K, newK);
    d[0].count = (int64_t)(xy.size() / 2);
    d[0].src = d[0].dst = xy.data();
    undistort_point_sets(d);
}

void Line3D::undistortSegments(std::vector<Vec4f>& segs, const LensDistortion& lens, const Matrix3d& K, const Matrix3d& newK)
{
    std::vector<l3d_points_desc> d(1);
    d[0].cam = lens_desc(lens, K, newK);
    d[0].count = 2 * (int64_t)segs.size();
    d[0].src = d[0].dst = segs.empty() ? nullptr : &segs[0].v[0];
    undistort_point_sets(d);
}

void Line3D::undistortPoints(std::vector<std::vector<float> >& xy, const std::vector<LensDistortion>& lenses, const std::vector<Matrix3d>& K,
                             const std::vector<Matrix3d>& newK)
{
    if (lenses.size() != xy.size() || K.size() != xy.size() || (!newK.empty() && newK.size() != xy.size()))
        throw std::invalid_argument("undistortPoints: one lens and one K (and one new K, if any) per point set");
    std::vector<l3d_points_desc> d(xy.size());
    for (size_t i = 0; i < xy.size(); ++i) {
        if (xy[i].size() % 2) throw std::invalid_argument("undistortPoints: an odd number of coordinates in set " + std::to_string(i));
        d[i].cam = lens_desc(lenses[i], K[i], newK.empty() ? Matrix3d() : newK[i]);
        d[i].count = (int64_t)(xy[i].size() / 2);
        d[i].src = d[i].dst = xy[i].data();
    }
    undistort_point_sets(d);
}

bool poseNeighbors(const std::vector<PoseView>& views, unsigned int num_neighbors, std::vector<std::list<unsigned int> >& neighbors, std::string* error,
                   int gx, int gy, int cuda_device)
{
    auto fail = [&](const std::string& what) { if (error) *error = "poseNeighbors: " + what; return false; };
    if (views.size() > (size_t)L3D_POSE_MAX_VIEWS) return fail("more than L3D_POSE_MAX_VIEWS views");
    const int n = (int)views.size();
    std::vector<l3d_pose_view> d((size_t)n);
    for (int i = 0; i < n; ++i) {
        const PoseView& v = views[i];
        l3d_pose_view& q = d[i];
        memset(&q, 0, sizeof(q));
        q.cam_id = v.id; q.width = v.width; q.height = v.height;
        q.fx = v.K(0, 0); q.skew = v.K(0, 1); q.cx = v.K(0, 2); q.fy = v.K(1, 1); q.cy = v.K(1, 2);
        memcpy(q.R, v.R.m, sizeof(q.R));
        q.t[0] = v.t.x; q.t[1] = v.t.y; q.t[2] = v.t.z;
        q.median_depth = v.median_depth;
    }
    int prev = 0;
    if (cudaGetDevice(&prev) != cudaSuccess || cudaSetDevice(cuda_device) != cudaSuccess) return fail("no usable CUDA device");
    struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};
    l3d_ctx* ctx = nullptr;
    if (l3d_ctx_create(cuda_device, &ctx) != L3D_OK) return fail("no usable CUDA device");
    std::vector<int64_t> ptr((size_t)n + 1);
    std::vector<uint32_t> cams((size_t)n * std::min<size_t>(num_neighbors, n > 0 ? (size_t)n - 1 : 0));
    const long long rc = l3d_pose_neighbors(ctx, n, d.data(), gx, gy, num_neighbors, ptr.data(), cams.data(), (long long)cams.size(), nullptr, nullptr);
    const std::string msg = l3d_last_error(ctx);
    l3d_ctx_destroy(ctx);
    if (rc < 0) { if (error) *error = msg; return false; }
    neighbors.assign((size_t)n, std::list<unsigned int>());
    for (int i = 0; i < n; ++i) neighbors[i].assign(cams.begin() + ptr[i], cams.begin() + ptr[i + 1]);
    return true;
}

}  // namespace L3DPP

// ================================================================================================ C wrapper (include/l3dpp_capi.h)
// The header spells Line3D's C++ types in C: check that they are the same.
static_assert(std::is_same<L3DPP::Line3D::MatchExchangeFn, l3dpp_exchange_fn>::value, "l3dpp_exchange_fn differs from Line3D::MatchExchangeFn");
static_assert(sizeof(l3dpp_stats_block) == sizeof(L3DPP::Line3DStats), "l3dpp_stats_block differs from Line3DStats");
#define L3DPP_SAME_STAT(f) static_assert(offsetof(l3dpp_stats_block, f) == offsetof(L3DPP::Line3DStats, f) && \
                                         std::is_same<decltype(l3dpp_stats_block::f), decltype(L3DPP::Line3DStats::f)>::value, "l3dpp_stats_block::" #f);
L3DPP_SAME_STAT(view_pairs) L3DPP_SAME_STAT(pair_evaluations) L3DPP_SAME_STAT(matches_after_knn) L3DPP_SAME_STAT(estimates)
L3DPP_SAME_STAT(affinity_entries) L3DPP_SAME_STAT(affinity_rows) L3DPP_SAME_STAT(clusters_total) L3DPP_SAME_STAT(clusters_valid)
L3DPP_SAME_STAT(lines3D) L3DPP_SAME_STAT(collinear_entries) L3DPP_SAME_STAT(opt_iterations) L3DPP_SAME_STAT(ms_match) L3DPP_SAME_STAT(ms_score)
L3DPP_SAME_STAT(ms_affinity) L3DPP_SAME_STAT(ms_diffusion) L3DPP_SAME_STAT(ms_cluster) L3DPP_SAME_STAT(opt_cost_before)
L3DPP_SAME_STAT(opt_cost_after) L3DPP_SAME_STAT(ms_gather)
#undef L3DPP_SAME_STAT

extern "C" {
using namespace L3DPP;
void* l3dpp_create(const char* output_folder, int load_segments, int max_img_width, unsigned int max_line_segments, int neighbors_by_worldpoints,
                   int use_gpu, const int* devices, int num_devices)
{
    try {
        return new Line3D(output_folder, load_segments != 0, max_img_width, max_line_segments, neighbors_by_worldpoints != 0, use_gpu != 0,
                          std::vector<int>(devices, devices + std::max(num_devices, 0)));
    } catch (...) { return nullptr; }
}
void l3dpp_destroy(void* h) { delete (Line3D*)h; }
const char* l3dpp_last_error(void* h) { return ((Line3D*)h)->lastError(); }
void* l3dpp_ctx(void* h) { return ((Line3D*)h)->impl()->ctx; }
int l3dpp_add_image(void* h, unsigned int cam, int w, int hgt, const double* K, const double* R, const double* t, float median_depth,
                    const unsigned int* list, int nlist, const float* segs, int nseg)
{
    Matrix3d Km, Rm; memcpy(Km.m, K, 72); memcpy(Rm.m, R, 72);
    std::vector<Vec4f> s(nseg); if (nseg) memcpy(s.data(), segs, 16 * (size_t)nseg);
    Line3D* L = (Line3D*)h;
    return L->addImage(cam, w, hgt, Km, Rm, Vector3d(t[0], t[1], t[2]), median_depth, std::list<unsigned int>(list, list + nlist), s) ? 0 : -1;
}
int l3dpp_match_images(void* h, float sp, float sa, unsigned int nn, float epi, int knn, float crd)
{ Line3D* L = (Line3D*)h; L->matchImages(sp, sa, nn, epi, knn, crd); return L->lastError()[0] ? -1 : 0; }
int l3dpp_reconstruct_opt(void* h, unsigned int vis, int diffusion, float collin, int use_ceres, unsigned int max_iter)
{ Line3D* L = (Line3D*)h; L->reconstruct3Dlines(vis, diffusion != 0, collin, use_ceres != 0, max_iter); return L->lastError()[0] ? -1 : 0; }
int l3dpp_set_line_candidates(void* h, unsigned int cam_a, unsigned int cam_b, const unsigned int* seg_pairs, long long n)
{
    Line3D* L = (Line3D*)h;
    if (n < 0 || (n > 0 && !seg_pairs)) { L->impl()->fail("setLineCandidates: n < 0, or no correspondence array for n > 0"); return -1; }
    std::vector<std::pair<unsigned int, unsigned int> > v((size_t)n);
    for (size_t i = 0; i < v.size(); ++i) v[i] = std::make_pair(seg_pairs[2 * i], seg_pairs[2 * i + 1]);
    L->setLineCandidates(cam_a, cam_b, v);
    return L->lastError()[0] ? -1 : 0;
}
int l3dpp_clear_line_candidates(void* h) { Line3D* L = (Line3D*)h; L->clearLineCandidates(); return L->lastError()[0] ? -1 : 0; }
int l3dpp_set_shard(void* h, int rank, int world, l3dpp_exchange_fn fn, void* user)
{ Line3D* L = (Line3D*)h; L->setShard(rank, world, fn, user); return L->lastError()[0] ? -1 : 0; }
int l3dpp_stats(void* h, l3dpp_stats_block* out) { memcpy(out, &((Line3D*)h)->stats(), sizeof(*out)); return 0; }
int l3dpp_view_index(void* h, unsigned int cam) { auto& m = ((Line3D*)h)->impl()->index_of; auto it = m.find(cam); return it == m.end() ? -1 : it->second; }
int l3dpp_collinear_from_cluster(void* h, const double* p1p2, int nres, const unsigned int* cams, const unsigned int* segs, double* out6, int cap)
{
    Line3D::Impl& P = *((Line3D*)h)->impl();
    if (P.vlist.size() != P.views.size()) { P.index_views(); P.matched = false; }   // as matchImages does, which outdates its results
    std::list<Segment2D> res;
    for (int i = 0; i < nres; ++i) res.push_back(Segment2D(cams[i], segs[i]));
    const LineCluster3D cl(Segment3D(Vector3d(p1p2[0], p1p2[1], p1p2[2]), Vector3d(p1p2[3], p1p2[4], p1p2[5])), res, nres ? cams[0] : 0);
    int n = 0;
    for (const Segment3D& sg : P.collinear_segments(cl)) {
        if (n < cap) { double* o = out6 + 6 * n; o[0] = sg.P1().x; o[1] = sg.P1().y; o[2] = sg.P1().z; o[3] = sg.P2().x; o[4] = sg.P2().y; o[5] = sg.P2().z; }
        ++n;
    }
    return n;
}
int l3dpp_view_info(void* h, unsigned int cam, float* k, float* md)
{ auto& v = ((Line3D*)h)->impl()->views; auto it = v.find(cam); if (it == v.end()) return -1; *k = it->second.k; *md = it->second.median_depth; return 0; }
int l3dpp_get_pairs(void* h, int* out, int cap)
{
    Line3D::Impl* P = ((Line3D*)h)->impl();
    const int n = (int)(P->pairs.size() / 2);
    for (int i = 0; i < n && i < cap; ++i) { out[2 * i] = (int)P->vlist[P->pairs[2 * i]]->id; out[2 * i + 1] = (int)P->vlist[P->pairs[2 * i + 1]]->id; }
    return n;
}
long long l3dpp_get_affinity(void* h, int raw, int* ei, int* ej, float* ew, long long cap)
{
    Line3D::Impl* P = ((Line3D*)h)->impl();
    const L3DPP::Affinity& A = raw ? P->A_raw : P->A;
    for (size_t e = 0; e < A.w.size() && (long long)e < cap; ++e) { ei[e] = A.i[e]; ej[e] = A.j[e]; ew[e] = A.w[e]; }
    return (long long)A.w.size();
}
int l3dpp_get_local2global(void* h, unsigned int* cam_seg, int cap)
{
    Line3D::Impl* P = ((Line3D*)h)->impl();
    for (size_t i = 0; i < P->local2global.size() && (int)i < cap; ++i) { const Segment2D s = P->seg_of(P->local2global[i]); cam_seg[2 * i] = s.camID(); cam_seg[2 * i + 1] = s.segID(); }
    return (int)P->local2global.size();
}
long long l3dpp_get_segments3d(void* h, l3dpp_seg3d* out, long long cap)
{
    std::vector<FinalLine3D> L; ((Line3D*)h)->get3Dlines(L);
    long long n = 0;
    for (size_t i = 0; i < L.size(); ++i)
        for (const Segment3D& s : L[i].collinear3Dsegments_) {
            if (out && n < cap) { out[n].line = (int)i; out[n].pad = 0; out[n].p1[0] = s.P1().x; out[n].p1[1] = s.P1().y; out[n].p1[2] = s.P1().z; out[n].p2[0] = s.P2().x; out[n].p2[1] = s.P2().y; out[n].p2[2] = s.P2().z; }
            ++n;
        }
    return n;
}
long long l3dpp_get_residuals(void* h, l3dpp_residual* out, long long cap)
{
    std::vector<FinalLine3D> L; ((Line3D*)h)->get3Dlines(L);
    long long n = 0;
    for (size_t i = 0; i < L.size(); ++i)
        for (const Segment2D& s : *L[i].underlyingCluster_.residuals()) { if (out && n < cap) { out[n].line = (int)i; out[n].cam = s.camID(); out[n].seg = s.segID(); } ++n; }
    return n;
}
void* l3dpp_lines_handle(void* h) { std::vector<FinalLine3D>* v = new std::vector<FinalLine3D>(); ((Line3D*)h)->get3Dlines(*v); return v; }
int l3dpp_save_obj(void* h, const char* folder) { Line3D* L = (Line3D*)h; L->saveResultAsOBJ(folder); return L->lastError()[0] ? -1 : 0; }
int l3dpp_save_stl(void* h, const char* folder) { Line3D* L = (Line3D*)h; L->saveResultAsSTL(folder); return L->lastError()[0] ? -1 : 0; }
int l3dpp_output_filename(void* h, char* buf, int cap)
{ const std::string s = ((Line3D*)h)->createOutputFilename(); if ((int)s.size() + 1 > cap) return -1; memcpy(buf, s.c_str(), s.size() + 1); return (int)s.size(); }
int l3dpp_set_lines(void* h, int nlines, const int* nseg, const double* segs6, const int* nres, const unsigned int* res_cam, const unsigned int* res_seg)
{
    Line3D::Impl& P = *((Line3D*)h)->impl();
    std::lock_guard<std::mutex> g(P.mtx);
    P.lines3D.clear();
    size_t so = 0, ro = 0;
    for (int i = 0; i < nlines; ++i) {
        FinalLine3D f;
        for (int k = 0; k < nseg[i]; ++k, ++so) {
            const double* q = segs6 + 6 * so;
            f.collinear3Dsegments_.push_back(Segment3D(Vector3d(q[0], q[1], q[2]), Vector3d(q[3], q[4], q[5])));
        }
        std::list<Segment2D> res;
        for (int k = 0; k < nres[i]; ++k, ++ro) res.push_back(Segment2D(res_cam[ro], res_seg[ro]));
        f.underlyingCluster_ = LineCluster3D(f.collinear3Dsegments_.empty() ? Segment3D() : f.collinear3Dsegments_.front(), res, nres[i] ? res.front().camID() : 0);
        P.lines3D.push_back(f);
    }
    return 0;
}
int l3dpp_save_txt(void* h, const char* folder) { Line3D* L = (Line3D*)h; L->save3DLinesAsTXT(folder); return L->lastError()[0] ? -1 : 0; }
int l3dpp_save_bin(void* h, const char* folder) { Line3D* L = (Line3D*)h; L->save3DLinesAsBIN(folder); return L->lastError()[0] ? -1 : 0; }
int l3dpp_add_image_pixels(void* h, unsigned int cam, const unsigned char* pixels, int rows, int cols, int channels, long long step, const double* K,
                           const double* R, const double* t, float median_depth, const unsigned int* list, int nlist, const float* segs, int nseg)
{
    Image8u img(rows, cols, channels);
    const size_t row = (size_t)std::max(cols, 0) * std::max(channels, 0);
    for (int r = 0; r < rows && row; ++r) memcpy(img.data.data() + r * row, pixels + r * step, row);
    Matrix3d Km, Rm; memcpy(Km.m, K, 72); memcpy(Rm.m, R, 72);
    std::vector<Vec4f> s(nseg); if (nseg) memcpy(s.data(), segs, 16 * (size_t)nseg);
    Line3D* L = (Line3D*)h;
    return L->addImage(cam, img, Km, Rm, Vector3d(t[0], t[1], t[2]), median_depth, std::list<unsigned int>(list, list + nlist), s) ? 0 : -1;
}
// L3DPP::LensDistortion from its 9 doubles: model, k[6], p[2]
static LensDistortion lens_of(const double* lens9)
{
    LensDistortion lens;
    lens.model = (int)lens9[0];
    for (int k = 0; k < 6; ++k) lens.k[k] = lens9[1 + k];
    lens.p[0] = lens9[7]; lens.p[1] = lens9[8];
    return lens;
}
int l3dpp_add_image_lens(void* h, unsigned int cam, int w, int hgt, const double* K, const double* R, const double* t, float median_depth,
                         const unsigned int* list, int nlist, const double* lens9, const float* segs, int nseg)
{
    Matrix3d Km, Rm; memcpy(Km.m, K, 72); memcpy(Rm.m, R, 72);
    std::vector<Vec4f> s(nseg); if (nseg) memcpy(s.data(), segs, 16 * (size_t)nseg);
    Line3D* L = (Line3D*)h;
    return L->addImage(cam, w, hgt, Km, Rm, Vector3d(t[0], t[1], t[2]), median_depth, std::list<unsigned int>(list, list + nlist), lens_of(lens9), s) ? 0 : -1;
}
int l3dpp_add_image_pixels_lens(void* h, unsigned int cam, const unsigned char* pixels, int rows, int cols, int channels, long long step,
                                const double* K, const double* R, const double* t, float median_depth, const unsigned int* list, int nlist,
                                const double* lens9, const float* segs, int nseg)
{
    Image8u img(rows, cols, channels);
    const size_t row = (size_t)std::max(cols, 0) * std::max(channels, 0);
    for (int r = 0; r < rows && row; ++r) memcpy(img.data.data() + r * row, pixels + r * step, row);
    Matrix3d Km, Rm; memcpy(Km.m, K, 72); memcpy(Rm.m, R, 72);
    std::vector<Vec4f> s(nseg); if (nseg) memcpy(s.data(), segs, 16 * (size_t)nseg);
    Line3D* L = (Line3D*)h;
    return L->addImage(cam, img, Km, Rm, Vector3d(t[0], t[1], t[2]), median_depth, std::list<unsigned int>(list, list + nlist), lens_of(lens9), s) ? 0 : -1;
}
int l3dpp_undistort_points(float* xy, const long long* counts, int n, const double* lens9, const double* K, const double* newK, int device, char* err,
                           int errcap)
{
    auto fail = [&](int rc, const char* what) { if (err && errcap > 0) snprintf(err, (size_t)errcap, "%s", what); return rc; };
    if (n < 0) return fail(-1, "undistortPoints: n < 0");
    int prev = 0;
    if (cudaGetDevice(&prev) != cudaSuccess || cudaSetDevice(device) != cudaSuccess) return fail(-2, "undistortPoints: no usable CUDA device");
    struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};
    std::vector<std::vector<float> > sets((size_t)n);
    std::vector<LensDistortion> lenses((size_t)n);
    std::vector<Matrix3d> Ks((size_t)n), newKs(newK ? (size_t)n : 0);
    size_t off = 0;
    for (int i = 0; i < n; ++i) {
        if (counts[i] < 0) return fail(-1, "undistortPoints: a negative count");
        sets[i].assign(xy + off, xy + off + 2 * (size_t)counts[i]);
        off += 2 * (size_t)counts[i];
        lenses[i] = lens_of(lens9 + 9 * i);
        memcpy(Ks[i].m, K + 9 * i, 72);
        if (newK) memcpy(newKs[i].m, newK + 9 * i, 72);
    }
    try {
        Line3D::undistortPoints(sets, lenses, Ks, newKs);
    } catch (const std::invalid_argument& e) { return fail(-1, e.what()); } catch (const std::exception& e) { return fail(-2, e.what()); }
    off = 0;
    for (int i = 0; i < n; ++i) { if (!sets[i].empty()) memcpy(xy + off, sets[i].data(), 4 * sets[i].size()); off += sets[i].size(); }
    return fail(0, "");
}
void l3dpp_push_detections(void* out, const float* xy4, long long n)
{
    std::vector<Vec4f>& v = *(std::vector<Vec4f>*)out;
    const size_t k = v.size();
    v.resize(k + (size_t)std::max(n, 0ll));
    if (n > 0) memcpy(v.data() + k, xy4, 16 * (size_t)n);
}
static bool l3dpp_detect_trampoline(void* user, const Image8u& gray, std::vector<Vec4f>& detections)
{
    const Line3D::Impl& P = *(const Line3D::Impl*)user;
    return P.c_detector.fn(P.c_detector.user, gray.data.data(), gray.rows, gray.cols, &detections) != 0;
}
int l3dpp_set_segment_detector(void* h, l3dpp_detect_fn fn, void* user)
{
    Line3D* L = (Line3D*)h;
    Line3D::Impl& P = *L->impl();
    { std::lock_guard<std::mutex> g(P.mtx); P.c_detector.fn = fn; P.c_detector.user = user; }
    L->setSegmentDetector(fn ? l3dpp_detect_trampoline : nullptr, &P);
    return 0;
}
long long l3dpp_view_segments(void* h, unsigned int cam, float* out, long long cap)
{
    Line3D* L = (Line3D*)h;
    long long n;
    {
        Line3D::Impl& P = *L->impl();
        std::lock_guard<std::mutex> g(P.mtx);
        auto it = P.views.find(cam);
        if (it == P.views.end()) return -1;
        n = (long long)it->second.lines.size();
    }
    for (long long i = 0; i < n && i < cap; ++i) memcpy(out + 4 * i, L->getSegmentCoords2D(cam, (unsigned int)i).v, 16);
    return n;
}
long long l3dpp_filter_detections(const float* det, long long n, int w, int h, int w_p, int h_p, unsigned int max_segments, float* out, long long cap)
{
    std::vector<Vec4f> d((size_t)std::max(n, 0ll));
    if (n > 0) memcpy(d.data(), det, 16 * (size_t)n);
    const std::vector<Vec4f> r = filter_detections(d, w, h, w_p, h_p, max_segments);
    if ((long long)r.size() <= cap && !r.empty()) memcpy(out, r.data(), 16 * r.size());
    return (long long)r.size();
}
int l3dpp_undistort_image(const unsigned char* src, unsigned char* dst, int rows, int cols, int channels, const double* radial, const double* tangential,
                          const double* K)
{
    Image8u in(rows, cols, channels), out;
    if (!in.data.empty()) memcpy(in.data.data(), src, in.data.size());
    Matrix3d Km; memcpy(Km.m, K, 72);
    try {
        Line3D::undistortImage(in, out, Vector3d(radial[0], radial[1], radial[2]), Vector2d(tangential[0], tangential[1]), Km);
    } catch (const std::invalid_argument&) { return -1; } catch (const std::exception&) { return -2; }
    memcpy(dst, out.data.data(), out.data.size());
    return 0;
}
int l3dpp_undistort_image_lens(const unsigned char* src, unsigned char* dst, int rows, int cols, int channels, const double* lens9, const double* K,
                               int device)
{
    const double zero[9] = {};
    return l3dpp_undistort_image_newk(src, dst, rows, cols, channels, lens9, K, zero, 0, 0, device);
}
int l3dpp_undistort_image_newk(const unsigned char* src, unsigned char* dst, int rows, int cols, int channels, const double* lens9, const double* K,
                               const double* newK, int out_rows, int out_cols, int device)
{
    int prev = 0;
    if (cudaGetDevice(&prev) != cudaSuccess || cudaSetDevice(device) != cudaSuccess) return -2;
    struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};
    Image8u in(rows, cols, channels), out;
    if (!in.data.empty()) memcpy(in.data.data(), src, in.data.size());
    Matrix3d Km, nKm; memcpy(Km.m, K, 72); memcpy(nKm.m, newK, 72);
    LensDistortion lens;
    lens.model = (int)lens9[0];
    for (int k = 0; k < 6; ++k) lens.k[k] = lens9[1 + k];
    lens.p[0] = lens9[7]; lens.p[1] = lens9[8];
    try {
        Line3D::undistortImage(in, out, lens, Km, nKm, out_cols, out_rows);
    } catch (const std::invalid_argument&) { return -1; } catch (const std::exception&) { return -2; }
    memcpy(dst, out.data.data(), out.data.size());
    return 0;
}
}
