// oracle/l3d_oracle.cc — CPU ORACLE for the Line3D++ matching / scoring / affinity / diffusion / clustering path.
//
// TEST INFRASTRUCTURE ONLY (see l3d_oracle.h).  A plain, single-threaded-by-default C++ restatement of what the
// reference computes, every function citing the reference file:line it follows (paths relative to /root/reference).
// Build: g++ -O2 -ffp-contract=off (no FMA contraction, so the float "GPU emulation" functions perform exactly the
// IEEE operation sequence of the reference kernels compiled with nvcc -fmad=false).
//
// Two semantics, like the reference's use_GPU switch (line3D.cc:49-53, 708-757):
//   REF_GPU : float kernels of cudawrapper.cu emulated on the CPU (+ the host staging of matchingGPU/scoringGPU)
//   REF_CPU : matchingCPU / scoringCPU double-precision path
// Known, unavoidable CPU-vs-GPU differences of the emulation (documented in DESIGN.md): rsqrtf / expf / acosf are the
// host libm versions here, so depths/scores agree with the GPU to ~1e-6 relative, not bitwise.  `overlap` (only
// + - * / sqrt) IS bitwise reproducible and so is kNN membership.
#include "l3d_oracle.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <limits>
#include <list>
#include <map>
#include <queue>
#include <set>
#include <string>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

const double L3D_EPS = 1e-12;                 // commons.h:92
const float L3D_EPS_GPU = 1e-12;              // cudawrapper.h:50  (float!)
const float L3D_PI_1_32 = 0.098174771f;       // commons.h:99
const float L3D_PI_31_32 = 3.043417886f;      // commons.h:100
const float MIN_SIMILARITY_3D = 0.50f;        // commons.h:58
const float MIN_BEST_SCORE_3D = 0.75f;        // commons.h:59
const float MIN_BEST_SCORE_PERC = 0.10f;      // commons.h:60
const float MIN_AFFINITY = 0.50f;             // commons.h:68
const int RDD_MAX_ITER = 10;                  // commons.h:65
const double PI_D = 3.14159265358979323846;   // CUDART_PI (math_constants.h:111) == M_PI
int g_threads = 1;

// ------------------------------------------------------------------------------------------------ float3 helpers
struct f3 { float x, y, z; };
struct f4 { float x, y, z, w; };
inline f3 mk3(float x, float y, float z) { f3 r = {x, y, z}; return r; }
inline f3 sub(f3 a, f3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }                 // helper_math.h:579
inline f3 add(f3 a, f3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }                 // helper_math.h:349
inline f3 scale(f3 a, float b) { return mk3(a.x * b, a.y * b, a.z * b); }                  // helper_math.h:814
inline float dot3(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }                // helper_math.h:1248
inline f3 cross3(f3 a, f3 b)                                                              // helper_math.h:1420
{ return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
inline float length3(f3 v) { return sqrtf(dot3(v, v)); }                                   // helper_math.h:1291
inline f3 normalize3(f3 v) { float inv = 1.0f / sqrtf(dot3(v, v)); return scale(v, inv); } // helper_math.h:1309 (rsqrtf)

// D_mult_matrix_vector_3, transpose=false (cudawrapper.cu:56-75); m is row-major 3x3
inline f3 mulmat(const float* m, f3 v)
{
    float o[3];
    for (int r = 0; r < 3; ++r) {
        o[r] = 0.0f;
        o[r] += m[r * 3 + 0] * v.x;
        o[r] += m[r * 3 + 1] * v.y;
        o[r] += m[r * 3 + 2] * v.z;
    }
    return mk3(o[0], o[1], o[2]);
}
// D_normalize_hom_coords_2D (cudawrapper.cu:18-30)
inline f3 normalize_hom(f3 p)
{
    if (fabsf(p.z) > L3D_EPS_GPU) { p.x /= p.z; p.y /= p.z; p.z /= p.z; p.z = 1; return p; }
    return mk3(0, 0, 0);
}
// D_point_on_segment_2D_f3 (cudawrapper.cu:80-86)
inline bool on_seg(f3 p1, f3 p2, f3 q)
{
    float v1x = p1.x - q.x, v1y = p1.y - q.y, v2x = p2.x - q.x, v2y = p2.y - q.y;
    return (v1x * v2x + v1y * v2y) < L3D_EPS_GPU;
}
// D_segment_overlap_2D (cudawrapper.cu:89-136)
inline float segment_overlap(f3 src_p1, f3 src_p2, f3 proj_q1, f3 proj_q2)
{
    float len_src = length3(sub(src_p1, src_p2));
    float len_tgt = length3(sub(proj_q1, proj_q2));
    if (len_src < 1.0f || len_tgt < 1.0f) return 0.0f;
    if (on_seg(src_p1, src_p2, proj_q1) && on_seg(src_p1, src_p2, proj_q2)) return len_tgt / len_src;
    else if (on_seg(proj_q1, proj_q2, src_p1) && on_seg(proj_q1, proj_q2, src_p2)) return len_src / len_tgt;
    else if (on_seg(src_p1, src_p2, proj_q1)) {
        float len1 = length3(sub(src_p2, proj_q2));
        float len2 = length3(sub(src_p1, proj_q2));
        if (on_seg(proj_q1, proj_q2, src_p1) && len1 > 1.0f) return length3(sub(proj_q1, src_p1)) / len1;
        else if (len2 > 1.0f) return length3(sub(proj_q1, src_p2)) / len2;
    } else if (on_seg(src_p1, src_p2, proj_q2)) {
        float len1 = length3(sub(src_p1, proj_q1));
        float len2 = length3(sub(src_p2, proj_q1));
        if (on_seg(proj_q1, proj_q2, src_p2) && len1 > 1.0f) return length3(sub(proj_q2, src_p2)) / len1;
        else if (len2 > 1.0f) return length3(sub(proj_q2, src_p1)) / len2;
    }
    return 0.0f;
}
// D_triangulate_depth (cudawrapper.cu:139-164)
inline void triangulate(f3 p1, f3 p2, f3 q1, f3 q2, f3 C_src, f3 C_tgt, const float* R_src, const float* R_tgt,
                        float* d1o, float* d2o)
{
    *d1o = -1; *d2o = -1;
    f3 ray_p1 = normalize3(mulmat(R_src, p1));
    f3 ray_p2 = normalize3(mulmat(R_src, p2));
    f3 ray_q1 = normalize3(mulmat(R_tgt, q1));
    f3 ray_q2 = normalize3(mulmat(R_tgt, q2));
    f3 n = normalize3(cross3(ray_q1, ray_q2));
    float dotp1 = dot3(n, ray_p1), dotp2 = dot3(n, ray_p2);
    if (fabsf(dotp1) < L3D_EPS_GPU || fabsf(dotp2) < L3D_EPS_GPU) return;
    *d1o = (dot3(C_tgt, n) - dot3(n, C_src)) / dotp1;
    *d2o = (dot3(C_tgt, n) - dot3(n, C_src)) / dotp2;
}
// body of K_match_lines for one (src y, tgt x) cell (cudawrapper.cu:198-252)
inline void match_cell(f4 ls, f4 lt, const float* F, const float* Rs, const float* Rt, f3 Cs, f3 Ct, float epi,
                       float* depths4, float* overlap_out)
{
    depths4[0] = depths4[1] = depths4[2] = depths4[3] = -1;
    f3 p1 = mk3(ls.x, ls.y, 1.0f), p2 = mk3(ls.z, ls.w, 1.0f);
    f3 q1 = mk3(lt.x, lt.y, 1.0f), q2 = mk3(lt.z, lt.w, 1.0f);
    f3 l_tgt = cross3(q1, q2);
    f3 epi_p1 = mulmat(F, p1), epi_p2 = mulmat(F, p2);
    f3 l2_p1 = normalize_hom(cross3(l_tgt, epi_p1));
    f3 l2_p2 = normalize_hom(cross3(l_tgt, epi_p2));
    if (int(l2_p1.z) == 0 || int(l2_p2.z) == 0) { *overlap_out = 0.0f; return; }
    float overlap = segment_overlap(q1, q2, l2_p1, l2_p2);
    if (overlap > epi) {
        triangulate(p1, p2, q1, q2, Cs, Ct, Rs, Rt, &depths4[0], &depths4[1]);
        triangulate(q1, q2, p1, p2, Ct, Cs, Rt, Rs, &depths4[2], &depths4[3]);
    }
    *overlap_out = overlap;
}

// Match_kNN comparator + pairwise_matches queue (commons.h:217-228)
struct MatchKNN { bool operator()(const orc_match_t& a, const orc_match_t& b) const { return a.overlap < b.overlap; } };
typedef std::priority_queue<orc_match_t, std::vector<orc_match_t>, MatchKNN> knn_queue;

// ------------------------------------------------------------------------------------------------ double helpers
struct V3 { double x, y, z; };
inline V3 V(double x, double y, double z) { V3 r = {x, y, z}; return r; }
inline V3 operator+(V3 a, V3 b) { return V(a.x + b.x, a.y + b.y, a.z + b.z); }
inline V3 operator-(V3 a, V3 b) { return V(a.x - b.x, a.y - b.y, a.z - b.z); }
inline V3 operator*(V3 a, double s) { return V(a.x * s, a.y * s, a.z * s); }
inline double dotd(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline V3 crossd(V3 a, V3 b) { return V(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
inline double normd(V3 a) { return std::sqrt(dotd(a, a)); }
inline V3 normalized(V3 a) { double n2 = dotd(a, a); if (n2 > 0) { double n = std::sqrt(n2); return V(a.x / n, a.y / n, a.z / n); } return a; }
struct M3 { double m[9]; double& operator()(int r, int c) { return m[r * 3 + c]; } double operator()(int r, int c) const { return m[r * 3 + c]; } };
inline M3 mul(const M3& a, const M3& b)
{ M3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += a(i, k) * b(k, j); r(i, j) = s; } return r; }
inline V3 mul(const M3& a, V3 v)
{ return V(a(0, 0) * v.x + a(0, 1) * v.y + a(0, 2) * v.z, a(1, 0) * v.x + a(1, 1) * v.y + a(1, 2) * v.z, a(2, 0) * v.x + a(2, 1) * v.y + a(2, 2) * v.z); }
inline M3 transpose(const M3& a) { M3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r(i, j) = a(j, i); return r; }
inline M3 inverse(const M3& a)  // cofactor formula (what Eigen uses for fixed 3x3)
{
    M3 r;
    double c00 = a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1), c01 = a(1, 2) * a(2, 0) - a(1, 0) * a(2, 2), c02 = a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0);
    double det = a(0, 0) * c00 + a(0, 1) * c01 + a(0, 2) * c02;
    double id = 1.0 / det;
    r(0, 0) = c00 * id; r(1, 0) = c01 * id; r(2, 0) = c02 * id;
    r(0, 1) = (a(0, 2) * a(2, 1) - a(0, 1) * a(2, 2)) * id; r(1, 1) = (a(0, 0) * a(2, 2) - a(0, 2) * a(2, 0)) * id; r(2, 1) = (a(0, 1) * a(2, 0) - a(0, 0) * a(2, 1)) * id;
    r(0, 2) = (a(0, 1) * a(1, 2) - a(0, 2) * a(1, 1)) * id; r(1, 2) = (a(0, 2) * a(1, 0) - a(0, 0) * a(1, 2)) * id; r(2, 2) = (a(0, 0) * a(1, 1) - a(0, 1) * a(1, 0)) * id;
    return r;
}

// Segment3D (segment3D.h:35-94)
struct Seg3D {
    V3 P1, P2, dir; float length; bool valid;
    Seg3D() : P1(V(0, 0, 0)), P2(V(0, 0, 0)), dir(V(0, 0, 0)), length(0.0f), valid(false) {}
    Seg3D(V3 a, V3 b)
    {
        length = (float)normd(a - b);
        if (length > L3D_EPS) { P1 = a; P2 = b; dir = normalized(b - a); valid = true; }
        else { P1 = P2 = dir = V(0, 0, 0); length = 0.0f; valid = false; }
    }
    // distance_Point2Line (segment3D.h:69-73): P1 + (dir * (P-P1)^T) * dir, evaluated as outer product times vector
    float distance_Point2Line(V3 P) const
    {
        V3 w = P - P1;
        double d[3] = {dir.x, dir.y, dir.z}, ww[3] = {w.x, w.y, w.z}, h[3];
        for (int i = 0; i < 3; ++i) h[i] = (d[i] * ww[0]) * d[0] + (d[i] * ww[1]) * d[1] + (d[i] * ww[2]) * d[2];
        V3 hp = V(P1.x + h[0], P1.y + h[1], P1.z + h[2]);
        return (float)normd(hp - P);
    }
    void translate(V3 t) { P1 = P1 + t; P2 = P2 + t; }
};

struct Seg2D { uint32_t cam, seg; bool operator<(const Seg2D& o) const { return cam < o.cam || (cam == o.cam && seg < o.seg); } };

// View (view.h, view.cc)
struct View {
    uint32_t id; unsigned width, height;
    M3 K, R, Kinv, Rt, RtKinv; V3 t, C, pp;
    float C_f3[3], RtKinv_f[9];               // view.cc:35-40 (set once at construction: NOT updated by translate())
    float k, median_depth, median_sigma, initial_median_depth, diagonal, min_line_length;
    std::vector<f4> lines;
    float collin_t = 0.0f;                     // View::collin_t_ (view.cc:29)
    std::vector<std::list<uint32_t> > collin;  // View::collin_ (view.h), filled by findCollinGPU / findCollinCPU

    void init()                               // View::View view.cc:6-42
    {
        diagonal = sqrtf(float(width * width + height * height));
        min_line_length = diagonal * 0.005f;
        pp = V(K(0, 2), K(1, 2), 1.0);
        Kinv = inverse(K); Rt = transpose(R); RtKinv = mul(Rt, Kinv);
        C = mul(Rt, t * -1.0);
        k = 0.0f; median_depth = 0.0f; median_sigma = 0.0f;
        C_f3[0] = (float)C.x; C_f3[1] = (float)C.y; C_f3[2] = (float)C.z;
        for (int i = 0; i < 9; ++i) RtKinv_f[i] = (float)RtKinv.m[i];
    }
    V3 ray(V3 p) const { return normalized(mul(RtKinv, p)); }                         // view.cc:317-321
    float specificSpatialReg(float r) const                                          // view.cc:307-314
    {
        V3 pps = pp + V(r, 0.0, 0.0);
        double a = std::acos(std::fmin(std::fmax(dotd(ray(pp), ray(pps)), -1.0), 1.0));
        return (float)std::sin(a);
    }
    Seg3D unprojectSegment(uint32_t seg, float d1, float d2) const                   // view.cc:356-371
    {
        if (seg >= lines.size()) return Seg3D();
        V3 p1 = V(lines[seg].x, lines[seg].y, 1.0), p2 = V(lines[seg].z, lines[seg].w, 1.0);
        return Seg3D(C + ray(p1) * (double)d1, C + ray(p2) * (double)d2);
    }
    float regularizerFrom3Dpoint(V3 P) const { return (float)(normd(P - C) * (double)k); }   // view.cc:445-448
    double segmentQualityAngle(const Seg3D& s, uint32_t seg) const                   // view.cc:466-484
    {
        if (seg >= lines.size()) return 0.0;
        double px = 0.5 * ((double)lines[seg].x + (double)lines[seg].z), py = 0.5 * ((double)lines[seg].y + (double)lines[seg].w);
        V3 r1 = ray(V(px, py, 1.0));
        return std::acos(std::fmin(std::fmax(dotd(r1, s.dir), -1.0), 1.0));
    }
    void project(V3 P, double* u, double* v) const                                   // view.cc:374-393
    {
        V3 q = mul(R, P) + t;
        double xn = (1.0 * q.x + 0.0 * q.z) / q.z, yn = (1.0 * q.y + 0.0 * q.z) / q.z;
        V3 h = mul(K, V(xn, yn, 1));
        *u = h.x / h.z; *v = h.y / h.z;
    }
    bool projectedLongEnough(const Seg3D& s) const                                   // view.cc:423-428
    {
        double u1, v1, u2, v2; project(s.P1, &u1, &v1); project(s.P2, &u2, &v2);
        return std::sqrt((u1 - u2) * (u1 - u2) + (v1 - v2) * (v1 - v2)) > min_line_length;
    }
    void translate(V3 tr) { C = C + tr; t = mul(R, C) * -1.0; }                       // view.cc:510-514
    void update_median_depth(float d, float sigmaP, float med_scene_depth)           // view.h:108-121
    {
        median_depth = d;
        if (sigmaP > 0.0f) k = sigmaP / med_scene_depth;
        median_sigma = k * median_depth;
    }
    double opticalAxesAngle(const View& v) const { return std::acos(std::fmin(std::fmax(dotd(ray(pp), v.ray(v.pp)), -1.0), 1.0)); } // view.cc:457-463
    float distanceVisualNeighborScore(const View& v) const                           // view.cc:487-501
    { V3 c = mul(R, v.C) + t; return fabsf((float)c.x) + fabsf((float)c.y); }
    float baseLine(const View& v) const { return (float)normd(C - v.C); }             // view.cc:504-507
};

// ------------------------------------------------------------------------------------------------ kernel-level (stateless)

typedef long long (*match_lines_fn_t)(const float*, int, const float*, int, const float*, const float*, const float*,
                                      const float*, const float*, uint32_t, uint32_t, float, int, int*, orc_match_t*, int, double*);
typedef int (*score_matches_fn_t)(const float*, int, const float*, int, const int*, const float*, const float*, const float*,
                                  float, float, float, float*, float*);
typedef int (*rdd_fn_t)(int, const int*, const int*, const float*, int, int*, int*, float*, double*);

struct CLEdge { int i, j; float w; };  // clustering.h:47-51

// performClustering (clustering.cc:6-48) + CLUniverse (universe.h:49-104)
struct Universe {
    struct El { int rank, id, size; };
    std::vector<El> e; int num;
    explicit Universe(int n) : e(n), num(n) { for (int i = 0; i < n; ++i) { e[i].rank = 0; e[i].size = 1; e[i].id = i; } }
    int find(int x) { int y = x; while (y != e[y].id) y = e[y].id; e[x].id = y; return y; }
    void join(int x, int y)
    {
        if (e[x].rank > e[y].rank) { e[y].id = x; e[x].size += e[y].size; }
        else { e[x].id = y; e[y].size += e[x].size; if (e[x].rank == e[y].rank) e[y].rank++; }
        --num;
    }
};
Universe* perform_clustering(std::list<CLEdge>& edges, int n, float c)
{
    if (edges.empty()) return NULL;
    edges.sort([](const CLEdge& a, const CLEdge& b) { return a.w < b.w; });   // sortCLEdgesByWeight, stable
    Universe* u = new Universe(n);
    std::vector<float> thr(n, c);
    for (std::list<CLEdge>::const_iterator it = edges.begin(); it != edges.end(); ++it) {
        int a = u->find(it->i), b = u->find(it->j);
        if (a != b && it->w <= thr[a] && it->w <= thr[b]) {
            u->join(a, b);
            a = u->find(a);
            thr[a] = it->w + c / (float)u->e[a].size;
        }
    }
    return u;
}

// SparseMatrix ctor (sparsematrix.cc:8-61): sorted COO + start index per row/col (-1 if empty)
struct Sparse {
    std::vector<f4> e; std::vector<int> start; bool row_sorted;
};
void build_sparse(std::list<CLEdge> entries, int n, bool by_row, Sparse& S)
{
    if (by_row) entries.sort([](const CLEdge& a, const CLEdge& b) { return a.i < b.i || (a.i == b.i && a.j < b.j); });
    else entries.sort([](const CLEdge& a, const CLEdge& b) { return a.j < b.j || (a.j == b.j && a.i < b.i); });
    S.e.clear(); S.start.assign(n, -1); S.row_sorted = by_row;
    int pos = 0, cur = -1;
    for (std::list<CLEdge>::const_iterator it = entries.begin(); it != entries.end(); ++it, ++pos) {
        f4 v = {(float)it->i, (float)it->j, it->w / 1.0f, 0.0f};
        S.e.push_back(v);
        int rc = by_row ? it->i : it->j;
        if (cur != rc) { S.start[rc] = pos; cur = rc; }
    }
}
// K_sparseMat_row_normalization (cudawrapper.cu:432-477)
void rdd_row_normalize(Sparse& P)
{
    int nnz = (int)P.e.size();
    for (int y = 0; y < (int)P.start.size(); ++y) {
        int start = P.start[y];
        if (start < 0) continue;   // (the kernel would read data[-1]; cannot happen: every id has an edge)
        float sum = 0.0f; int i = start;
        while (i < nnz) { if ((int)P.e[i].x != y) break; sum += P.e[i].z; ++i; }
        if (sum < L3D_EPS_GPU) sum = L3D_EPS_GPU;
        i = start;
        while (i < nnz) { if ((int)P.e[i].x != y) break; P.e[i].z /= sum; ++i; }
    }
}
// K_sparseMat_diffusion_step (cudawrapper.cu:480-544)
void rdd_step(const Sparse& P, const Sparse& W, Sparse& Pp)
{
    int nnz = (int)P.e.size();
    for (int y = 0; y < nnz; ++y) {
        f4 data = P.e[y];
        int r = (int)data.y, c = (int)data.x;
        float mul = 0.0f;
        int sP = P.start[r], sW = W.start[c];
        while (sP >= 0 && sW >= 0 && sP < nnz && sW < nnz) {
            f4 d1 = P.e[sP], d2 = W.e[sW];
            if ((int)d1.x != r || (int)d2.y != c) break;
            mul += d1.z * d2.z;
            ++sP; ++sW;
        }
        mul *= data.z;
        if (mul < L3D_EPS_GPU) mul = L3D_EPS_GPU;
        int s = Pp.start[r];
        bool found = false;
        while (s >= 0 && s < nnz && !found) {
            if ((int)Pp.e[s].x != r) break;
            if ((int)Pp.e[s].y == c) { Pp.e[s].z = mul; found = true; }
            ++s;
        }
    }
}

// K_collinearity (cudawrapper.cu:370-429) for one ordered cell: l1 = lines[x], l2 = lines[y], x > y; float arithmetic,
// D_point_on_segment_2D_f3 (80-86), cross (helper_math.h:1420), D_distance_p2l_2D_f3 (34-37)
inline float dist_p2l_f(f3 line, f3 p) { return fabsf((line.x * p.x + line.y * p.y + line.z) / sqrtf(line.x * line.x + line.y * line.y)); }
inline unsigned char collinear_cell_f32(f4 l1, f4 l2, float dist_t)
{
    f3 p0 = mk3(l1.x, l1.y, 1.0f), p1 = mk3(l1.z, l1.w, 1.0f), q0 = mk3(l2.x, l2.y, 1.0f), q1 = mk3(l2.z, l2.w, 1.0f);
    if (on_seg(p0, p1, q0) || on_seg(p0, p1, q1) || on_seg(q0, q1, p0) || on_seg(q0, q1, p1)) return 0;
    f3 line1 = cross3(p0, p1), line2 = cross3(q0, q1);
    float d1 = fmaxf(dist_p2l_f(line1, q0), dist_p2l_f(line1, q1));
    float d2 = fmaxf(dist_p2l_f(line2, p0), dist_p2l_f(line2, p1));
    return fmaxf(d1, d2) < dist_t ? 1 : 0;
}
// View::findCollinCPU (view.cc:212-263) for one (r, c) cell: double geometry, float distances
// (View::distance_point2line_2D view.cc:266-269 returns float and takes sqrtf of the double sum; pointOnSegment 290-296)
inline bool on_seg_d(V3 p1, V3 p2, V3 x) { return ((p1.x - x.x) * (p2.x - x.x) + (p1.y - x.y) * (p2.y - x.y)) < L3D_EPS; }
inline float dist_p2l_d(V3 line, V3 p) { return (float)std::fabs((line.x * p.x + line.y * p.y + line.z) / sqrtf((float)(line.x * line.x + line.y * line.y))); }
inline unsigned char collinear_cell_f64(f4 l1, f4 l2, float dist_t)
{
    V3 p0 = V(l1.x, l1.y, 1.0f), p1 = V(l1.z, l1.w, 1.0f), q0 = V(l2.x, l2.y, 1.0f), q1 = V(l2.z, l2.w, 1.0f);
    V3 line1 = crossd(p0, p1), line2 = crossd(q0, q1);
    if (on_seg_d(p0, p1, q0) || on_seg_d(p0, p1, q1) || on_seg_d(q0, q1, p0) || on_seg_d(q0, q1, p1)) return 0;
    float d1 = fmaxf(dist_p2l_d(line1, q0), dist_p2l_d(line1, q1));
    float d2 = fmaxf(dist_p2l_d(line2, p0), dist_p2l_d(line2, p1));
    return fmaxf(d1, d2) < dist_t ? 1 : 0;
}

typedef int (*collinear_fn_t)(const float*, int, float, unsigned char*, float*);

} // namespace

extern "C" {

void orc_set_threads(int n) { g_threads = n < 1 ? 1 : n; }

// find_collinear_segments_GPU (cudawrapper.cu:689-705) + K_collinearity: dense N x N char matrix, C[y*N+x]; the kernel
// evaluates the cells x >= y with l1 = lines[x], l2 = lines[y] and mirrors them (cudawrapper.cu:376-427)
int orc_collinear_f32(const float* lines, int N, float dist_t, unsigned char* C_out, float* kernel_ms)
{
    auto t0 = std::chrono::steady_clock::now();
    const f4* L = (const f4*)lines;
#pragma omp parallel for num_threads(g_threads) schedule(dynamic, 16)
    for (int y = 0; y < N; ++y)
        for (int x = y; x < N; ++x) {
            unsigned char v = x == y ? 0 : collinear_cell_f32(L[x], L[y], dist_t);
            C_out[(size_t)y * N + x] = v; C_out[(size_t)x * N + y] = v;
        }
    if (kernel_ms) *kernel_ms = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}
// View::findCollinCPU (view.cc:212-263) written as the same dense matrix: C[r*N+c] = 1 iff c is pushed to collin_[r]
int orc_collinear_f64(const float* lines, int N, float dist_t, unsigned char* C_out, float* kernel_ms)
{
    auto t0 = std::chrono::steady_clock::now();
    const f4* L = (const f4*)lines;
#pragma omp parallel for num_threads(g_threads) schedule(static)
    for (int r = 0; r < N; ++r)
        for (int c2 = 0; c2 < N; ++c2)
            C_out[(size_t)r * N + c2] = r == c2 ? 0 : collinear_cell_f64(L[r], L[c2], dist_t);
    if (kernel_ms) *kernel_ms = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

int orc_match_dense_f32(const float* lines_src, int Ns, const float* lines_tgt, int Nt, const float* F,
                        const float* RtKinv_src, const float* RtKinv_tgt, const float* C_src, const float* C_tgt,
                        float epi_overlap, float* depths_out, float* overlaps_out, float* kernel_ms)
{
    auto t0 = std::chrono::steady_clock::now();
    f3 Cs = mk3(C_src[0], C_src[1], C_src[2]), Ct = mk3(C_tgt[0], C_tgt[1], C_tgt[2]);
#pragma omp parallel for num_threads(g_threads) schedule(static)
    for (int r = 0; r < Ns; ++r) {
        f4 ls = {lines_src[4 * r], lines_src[4 * r + 1], lines_src[4 * r + 2], lines_src[4 * r + 3]};
        for (int c = 0; c < Nt; ++c) {
            f4 lt = {lines_tgt[4 * c], lines_tgt[4 * c + 1], lines_tgt[4 * c + 2], lines_tgt[4 * c + 3]};
            size_t o = (size_t)r * Nt + c;
            match_cell(ls, lt, F, RtKinv_src, RtKinv_tgt, Cs, Ct, epi_overlap, depths_out + 4 * o, overlaps_out + o);
        }
    }
    if (kernel_ms) *kernel_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

// K_match_lines + host post-pass of match_lines_GPU (cudawrapper.cu:592-650) without materialising the dense buffer
long long orc_match_lines_f32(const float* lines_src, int Ns, const float* lines_tgt, int Nt, const float* F,
                              const float* RtKinv_src, const float* RtKinv_tgt, const float* C_src,
                              const float* C_tgt, uint32_t srcCamID, uint32_t tgtCamID, float epi_overlap, int kNN,
                              int* counts, orc_match_t* out, int cap, double* wall_ms)
{
    auto t0 = std::chrono::steady_clock::now();
    f3 Cs = mk3(C_src[0], C_src[1], C_src[2]), Ct = mk3(C_tgt[0], C_tgt[1], C_tgt[2]);
    long long total = 0;
#pragma omp parallel for num_threads(g_threads) schedule(dynamic, 16) reduction(+ : total)
    for (int r = 0; r < Ns; ++r) {
        f4 ls = {lines_src[4 * r], lines_src[4 * r + 1], lines_src[4 * r + 2], lines_src[4 * r + 3]};
        // storage reserved up front: letting the vector grow inside the parallel loop (as the reference's per-row
        // pairwise_matches does) serialises the threads on malloc and would understate the CPU baseline
        std::vector<orc_match_t> q_store; q_store.reserve(1024);
        knn_queue q(MatchKNN(), std::move(q_store));
        int n_new = 0;
        for (int c = 0; c < Nt; ++c) {
            f4 lt = {lines_tgt[4 * c], lines_tgt[4 * c + 1], lines_tgt[4 * c + 2], lines_tgt[4 * c + 3]};
            float d[4], ov;
            match_cell(ls, lt, F, RtKinv_src, RtKinv_tgt, Cs, Ct, epi_overlap, d, &ov);
            if (d[0] > 0.0f && d[1] > 0.0f && d[2] > 0.0f && d[3] > 0.0f) {   // cudawrapper.cu:605
                orc_match_t M = {srcCamID, (uint32_t)r, tgtCamID, (uint32_t)c, ov, 0.0f, d[0], d[1], d[2], d[3]};
                if (kNN > 0) q.push(M);
                else { if (out && n_new < cap) out[(size_t)r * cap + n_new] = M; ++n_new; }
            }
        }
        if (kNN > 0)
            while (n_new < kNN && !q.empty()) {
                if (out && n_new < cap) out[(size_t)r * cap + n_new] = q.top();
                q.pop(); ++n_new;
            }
        if (counts) counts[r] = n_new;
        total += n_new;
    }
    if (wall_ms) *wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return total;
}

// matchingCPU (line3D.cc:900-1015) + pointOnSegment 1077-1083 + mutualOverlap 1086-1165 + triangulationDepths 1168-1193
long long orc_match_lines_f64(const float* lines_src, int Ns, const float* lines_tgt, int Nt, const double* Fd,
                              const double* RtKinv_src, const double* RtKinv_tgt, const double* C_src,
                              const double* C_tgt, uint32_t srcCamID, uint32_t tgtCamID, float epi_overlap, int kNN,
                              int* counts, orc_match_t* out, int cap, double* wall_ms)
{
    auto t0 = std::chrono::steady_clock::now();
    M3 F, Rs, Rt; memcpy(F.m, Fd, 72); memcpy(Rs.m, RtKinv_src, 72); memcpy(Rt.m, RtKinv_tgt, 72);
    V3 C1 = V(C_src[0], C_src[1], C_src[2]), C2 = V(C_tgt[0], C_tgt[1], C_tgt[2]);
    long long total = 0;
    auto pointOnSegment = [](V3 x, V3 p1, V3 p2) { return ((p1.x - x.x) * (p2.x - x.x) + (p1.y - x.y) * (p2.y - x.y)) < L3D_EPS; };
    auto tri = [](const M3& Rsrc, V3 Csrc, V3 p1, V3 p2, const M3& Rtgt, V3 Ctgt, V3 q1, V3 q2, double* d1, double* d2) {
        V3 ray_p1 = normalized(mul(Rsrc, p1)), ray_p2 = normalized(mul(Rsrc, p2));
        V3 ray_q1 = normalized(mul(Rtgt, q1)), ray_q2 = normalized(mul(Rtgt, q2));
        V3 n = normalized(crossd(ray_q1, ray_q2));
        if (std::fabs(dotd(ray_p1, n)) < L3D_EPS || std::fabs(dotd(ray_p2, n)) < L3D_EPS) { *d1 = -1; *d2 = -1; return; }
        *d1 = (dotd(Ctgt, n) - dotd(n, Csrc)) / dotd(n, ray_p1);
        *d2 = (dotd(Ctgt, n) - dotd(n, Csrc)) / dotd(n, ray_p2);
    };
#pragma omp parallel for num_threads(g_threads) schedule(dynamic, 16) reduction(+ : total)
    for (int r = 0; r < Ns; ++r) {
        int n_new = 0;
        V3 p1 = V(lines_src[4 * r], lines_src[4 * r + 1], 1.0), p2 = V(lines_src[4 * r + 2], lines_src[4 * r + 3], 1.0);
        V3 epi_p1 = mul(F, p1), epi_p2 = mul(F, p2);
        // storage reserved up front: letting the vector grow inside the parallel loop (as the reference's per-row
        // pairwise_matches does) serialises the threads on malloc and would understate the CPU baseline
        std::vector<orc_match_t> q_store; q_store.reserve(1024);
        knn_queue q(MatchKNN(), std::move(q_store));
        for (int c = 0; c < Nt; ++c) {
            V3 q1 = V(lines_tgt[4 * c], lines_tgt[4 * c + 1], 1.0), q2 = V(lines_tgt[4 * c + 2], lines_tgt[4 * c + 3], 1.0);
            V3 l2 = crossd(q1, q2);
            V3 p1p = crossd(l2, epi_p1), p2p = crossd(l2, epi_p2);
            if (std::fabs(p1p.z) > L3D_EPS && std::fabs(p2p.z) > L3D_EPS) {
                p1p = V(p1p.x / p1p.z, p1p.y / p1p.z, p1p.z / p1p.z);
                p2p = V(p2p.x / p2p.z, p2p.y / p2p.z, p2p.z / p2p.z);
                // mutualOverlap
                V3 cp[4] = {p1p, p2p, q1, q2};
                float score = 0.0f;
                if (pointOnSegment(cp[0], cp[2], cp[3]) || pointOnSegment(cp[1], cp[2], cp[3]) ||
                    pointOnSegment(cp[2], cp[0], cp[1]) || pointOnSegment(cp[3], cp[0], cp[1])) {
                    float max_dist = 0.0f; size_t o1 = 0, i1 = 1, i2 = 2, o2 = 3;
                    for (size_t i = 0; i < 3; ++i)
                        for (size_t j = i + 1; j < 4; ++j) {
                            float dist = (float)normd(cp[i] - cp[j]);
                            if (dist > max_dist) { max_dist = dist; o1 = i; o2 = j; }
                        }
                    if (max_dist < 1.0f) score = 0.0f;
                    else {
                        if (o1 == 0) { if (o2 == 1) { i1 = 2; i2 = 3; } else if (o2 == 2) { i1 = 1; i2 = 3; } else { i1 = 1; i2 = 2; } }
                        else if (o1 == 1) { i1 = 0; if (o2 == 2) i2 = 3; else i2 = 2; }
                        else { i1 = 0; i2 = 1; }
                        score = (float)(normd(cp[i1] - cp[i2]) / max_dist);
                    }
                }
                if (score > epi_overlap) {
                    double ds1, ds2, dt1, dt2;
                    tri(Rs, C1, p1, p2, Rt, C2, q1, q2, &ds1, &ds2);
                    tri(Rt, C2, q1, q2, Rs, C1, p1, p2, &dt1, &dt2);
                    if (ds1 > L3D_EPS && ds2 > L3D_EPS && dt1 > L3D_EPS && dt2 > L3D_EPS) {
                        orc_match_t M = {srcCamID, (uint32_t)r, tgtCamID, (uint32_t)c, score, 0.0f, (float)ds1, (float)ds2, (float)dt1, (float)dt2};
                        if (kNN > 0) q.push(M);
                        else { if (out && n_new < cap) out[(size_t)r * cap + n_new] = M; ++n_new; }
                    }
                }
            }
        }
        if (kNN > 0)
            while (n_new < kNN && !q.empty()) {
                if (out && n_new < cap) out[(size_t)r * cap + n_new] = q.top();
                q.pop(); ++n_new;
            }
        if (counts) counts[r] = n_new;
        total += n_new;
    }
    if (wall_ms) *wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return total;
}

// K_score_matches (cudawrapper.cu:256-367)
int orc_score_matches_f32(const float* lines, int Ns, const float* matches, int M, const int* ranges,
                          const float* reg_tgt, const float* RtKinv, const float* Cf, float two_sigA_sqr, float k,
                          float min_similarity, float* scores_out, float* kernel_ms)
{
    (void)Ns;
    auto t0 = std::chrono::steady_clock::now();
    f3 C = mk3(Cf[0], Cf[1], Cf[2]);
    auto unproject = [&](f3 p, float depth) { return add(C, scale(normalize3(mulmat(RtKinv, p)), depth)); };
    auto angle_deg = [](f3 v1, f3 v2) {
        float angle = (float)((double)acosf(fmaxf(fminf(dot3(v1, v2), 1.0f), -1.0f)) / PI_D * (double)180.0f);
        if (angle > 90.0f) angle = 180.0f - angle;
        return angle;
    };
#pragma omp parallel for num_threads(g_threads) schedule(dynamic, 64)
    for (int x = 0; x < M; ++x) {
        const float* m = matches + 4 * x;
        int tgt_cam_src = (int)m[1];
        float d1_src = m[2], d2_src = m[3];
        int lID = (int)m[0];
        f3 p1 = mk3(lines[4 * lID], lines[4 * lID + 1], 1.0f), p2 = mk3(lines[4 * lID + 2], lines[4 * lID + 3], 1.0f);
        f3 P1 = unproject(p1, d1_src), P2 = unproject(p2, d2_src);
        f3 dir_src = normalize3(sub(P2, P1));
        float sig1 = k * d1_src, sig2 = k * d2_src;
        float pos_reg1 = 2.0f * sig1 * sig1, pos_reg2 = 2.0f * sig2 * sig2;
        float pos_reg1_tgt = 2.0f * reg_tgt[2 * x] * reg_tgt[2 * x], pos_reg2_tgt = 2.0f * reg_tgt[2 * x + 1] * reg_tgt[2 * x + 1];
        pos_reg1 = 0.5f * (pos_reg1 + pos_reg1_tgt);
        pos_reg2 = 0.5f * (pos_reg2 + pos_reg2_tgt);
        int start = ranges[2 * lID], end = ranges[2 * lID + 1];
        float score3D = 0.0f; int current_cam = -1; float current_max_sim = 0.0f;
        for (int i = start; i <= end; ++i) {
            const float* m2 = matches + 4 * i;
            int tgt_cam_tgt = (int)m2[1];
            if (tgt_cam_src != tgt_cam_tgt) {
                float d1_tgt = m2[2], d2_tgt = m2[3];
                f3 Q1 = unproject(p1, d1_tgt), Q2 = unproject(p2, d2_tgt);
                f3 dir_tgt = normalize3(sub(Q2, Q1));
                float angle = angle_deg(dir_src, dir_tgt);
                float sim_a = expf(-angle * angle / two_sigA_sqr);
                float d1 = d1_src - d1_tgt, d2 = d2_src - d2_tgt;
                float sim_p1 = expf(-d1 * d1 / pos_reg1), sim_p2 = expf(-d2 * d2 / pos_reg2);
                float sim = fminf(sim_a, fminf(sim_p1, sim_p2));
                if (sim < min_similarity) sim = 0.0f;
                current_max_sim = fmaxf(current_max_sim, sim);
                if (current_cam != tgt_cam_tgt) { score3D += current_max_sim; current_max_sim = 0.0f; current_cam = tgt_cam_tgt; }
            }
        }
        score3D += current_max_sim;
        scores_out[x] = score3D;
    }
    if (kernel_ms) *kernel_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

// SparseMatrix(A_, n) + replicator_dynamics_diffusion_GPU (cudawrapper.cu:708-766) + download, with `iters` iterations
int orc_rdd_f32_iters(int nedges, const int* ei, const int* ej, const float* ew, int n, int iters, int* out_i, int* out_j,
                      float* out_w, double* wall_ms)
{
    auto t0 = std::chrono::steady_clock::now();
    std::list<CLEdge> A;
    for (int e = 0; e < nedges; ++e) { CLEdge ed = {ei[e], ej[e], ew[e]}; A.push_back(ed); }
    Sparse W, P, Pp;
    build_sparse(A, n, false, W);          // W col-sorted (default ctor args, sparsematrix.h)
    {   // SparseMatrix(W, true): re-sort copy by row (sparsematrix.cc:64-135)
        std::list<CLEdge> tmp;
        for (size_t i = 0; i < W.e.size(); ++i) { CLEdge ed = {(int)W.e[i].x, (int)W.e[i].y, W.e[i].z}; tmp.push_back(ed); }
        build_sparse(tmp, n, true, P);
    }
    Pp = P;                                // P_prime = copy of (un-normalised) P  cudawrapper.cu:724
    rdd_row_normalize(P);
    for (int it = 0; it < iters; ++it) {
        rdd_step(P, W, Pp);
        std::swap(P, Pp);
        if (it < iters - 1) rdd_row_normalize(P);
    }
    for (size_t i = 0; i < P.e.size(); ++i) { out_i[i] = (int)P.e[i].x; out_j[i] = (int)P.e[i].y; out_w[i] = P.e[i].z; }
    if (wall_ms) *wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}
// the reference's fixed iteration count (L3D_DEF_RDD_MAX_ITER); the signature of ref_rdd (rdd_fn_t)
int orc_rdd_f32(int nedges, const int* ei, const int* ej, const float* ew, int n, int* out_i, int* out_j,
                float* out_w, double* wall_ms)
{
    return orc_rdd_f32_iters(nedges, ei, ej, ew, n, RDD_MAX_ITER, out_i, out_j, out_w, wall_ms);
}

int orc_cluster(int nedges, const int* ei, const int* ej, const float* ew, int n, float c, int* labels_out)
{
    std::list<CLEdge> A;
    for (int e = 0; e < nedges; ++e) { CLEdge ed = {ei[e], ej[e], ew[e]}; A.push_back(ed); }
    Universe* u = perform_clustering(A, n, c);
    if (!u) return -1;
    for (int i = 0; i < n; ++i) labels_out[i] = u->find(i);
    delete u;
    return 0;
}

} // extern "C"

// ================================================================================================ line bundling
// LineOptimizer::optimize (optimization.cc:8-303) with LineReprojectionError (optimization.h:52-171).  The reference hands
// the problem to Ceres (third-party, NOT in /root/reference; CMake accepts any installed Ceres, CMakeLists.txt:120-134):
// cameras and intrinsics are set constant (optimization.cc:178-188), so only the 4 Cayley parameters of every line are
// free and the Jacobian is block diagonal (one 4-column block per line).  Restated here from Ceres' PUBLISHED algorithm
// (solver defaults of ceres-solver 1.13-2.1: trust_region_minimizer.cc, levenberg_marquardt_strategy.cc, corrector.cc,
// loss_function.cc): Levenberg-Marquardt trust region with ONE radius for the whole problem, Jacobi scaling fixed at
// iteration 0, Huber loss through the Triggs corrector, the function / gradient / parameter tolerances 1e-6 / 1e-10 /
// 1e-8, min_relative_decrease 1e-3, initial radius 1e4.  SPARSE_SCHUR on a block-diagonal system is a 4x4 Cholesky per
// line.  Exact derivatives by forward-mode dual numbers like ceres::AutoDiffCostFunction.
// Pinned against the reference's own before/after result fixtures (tests/golden/line3dpp_ref_opt_pairs_v1.npz).
namespace {

struct Jet4 { double a; double v[4]; };
inline Jet4 J(double a) { Jet4 r; r.a = a; r.v[0] = r.v[1] = r.v[2] = r.v[3] = 0.0; return r; }
inline Jet4 operator+(Jet4 x, Jet4 y) { Jet4 r; r.a = x.a + y.a; for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] + y.v[i]; return r; }
inline Jet4 operator-(Jet4 x, Jet4 y) { Jet4 r; r.a = x.a - y.a; for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] - y.v[i]; return r; }
inline Jet4 operator-(Jet4 x) { Jet4 r; r.a = -x.a; for (int i = 0; i < 4; ++i) r.v[i] = -x.v[i]; return r; }
inline Jet4 operator*(Jet4 x, Jet4 y) { Jet4 r; r.a = x.a * y.a; for (int i = 0; i < 4; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a; return r; }
inline Jet4 operator/(Jet4 x, Jet4 y)
{ Jet4 r; const double inv = 1.0 / y.a, q = x.a * inv; r.a = q; for (int i = 0; i < 4; ++i) r.v[i] = (x.v[i] - q * y.v[i]) * inv; return r; }
inline Jet4 operator*(double s, Jet4 x) { return J(s) * x; }
inline Jet4 operator*(Jet4 x, double s) { return x * J(s); }
inline Jet4 jsqrt(Jet4 x) { Jet4 r; r.a = std::sqrt(x.a); const double t = 1.0 / (2.0 * r.a); for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] * t; return r; }
inline Jet4 jacos(Jet4 x) { Jet4 r; r.a = std::acos(x.a); const double t = -1.0 / std::sqrt(1.0 - x.a * x.a); for (int i = 0; i < 4; ++i) r.v[i] = x.v[i] * t; return r; }
inline Jet4 jexp(Jet4 x) { Jet4 r; r.a = std::exp(x.a); for (int i = 0; i < 4; ++i) r.v[i] = r.a * x.v[i]; return r; }
inline bool jfinite(Jet4 x) { bool f = std::isfinite(x.a); for (int i = 0; i < 4; ++i) f = f && std::isfinite(x.v[i]); return f; }

struct OptCam { double R[9], C[3], fx, fy, px, py; };
struct OptObs { double x1, y1, x2, y2, nx, ny; };   // observed end points and NORMAL direction (-dir.y, dir.x), optimization.cc:160-166

// LineReprojectionError::operator() (optimization.h:66-162); line = (omega, sx, sy, sz).  AngleAxisRotatePoint(camera, m)
// with the angle-axis of R (optimization.cc:118-128) is R*m.
bool reprojection_error(const OptCam& cam, const OptObs& o, const Jet4 line[4], Jet4 res[2])
{
    const Jet4 omega = line[0], sx = line[1], sy = line[2], sz = line[3];
    const Jet4 nm = sx * sx + sy * sy + sz * sz;
    const Jet4 div = J(1.0) / (J(1.0) + nm);
    Jet4 l[3], m[3];
    l[0] = div * (J(1.0) - nm + J(2.0) * sx * sx);
    l[1] = div * (J(2.0) * sz + J(2.0) * sy * sx);
    l[2] = div * (J(-2.0) * sy + J(2.0) * sz * sx);
    m[0] = omega * div * (J(-2.0) * sz + J(2.0) * sx * sy);
    m[1] = omega * div * (J(1.0) - nm + J(2.0) * sy * sy);
    m[2] = omega * div * (J(2.0) * sx + J(2.0) * sz * sy);
    if (std::fabs(omega.a) < 1e-12) { res[0] = res[1] = J(0.0); return false; }
    Jet4 Ccl[3];
    Ccl[0] = cam.C[1] * l[2] - cam.C[2] * l[1];
    Ccl[1] = -(cam.C[0] * l[2] - cam.C[2] * l[0]);
    Ccl[2] = cam.C[0] * l[1] - cam.C[1] * l[0];
    m[0] = m[0] - Ccl[0]; m[1] = m[1] - Ccl[1]; m[2] = m[2] - Ccl[2];
    Jet4 q[3];
    for (int i = 0; i < 3; ++i) q[i] = cam.R[3 * i] * m[0] + cam.R[3 * i + 1] * m[1] + cam.R[3 * i + 2] * m[2];
    Jet4 pl[3];
    pl[0] = cam.fy * q[0];
    pl[1] = cam.fx * q[1];
    pl[2] = (-cam.fy * cam.px) * q[0] - (cam.fx * cam.py) * q[1] + (cam.fx * cam.fy) * q[2];
    const Jet4 d = jsqrt(pl[0] * pl[0] + pl[1] * pl[1]);
    if (d.a < 1e-12) { res[0] = res[1] = J(0.0); return false; }
    Jet4 aw = J(1.0);
    if (d.a > 1e-12) {
        const Jet4 dx = pl[0] / d, dy = pl[1] / d;
        const Jet4 dotp = dx * o.nx + dy * o.ny;
        Jet4 angle = jacos(dotp);
        if (jfinite(angle)) {
            if (angle.a > M_PI_2) angle = J(M_PI) - angle;
            aw = jexp(2.0 * angle);
        }
    }
    res[0] = (pl[0] * o.x1 + pl[1] * o.y1 + pl[2]) / d * aw;
    res[1] = (pl[0] * o.x2 + pl[1] * o.y2 + pl[2]) / d * aw;
    return true;
}

// 0.5 * sum rho(|r|^2) over the residual blocks of line i, its gradient g = J'r and H = J'J (robustified, UNscaled).
// HuberLoss(2) (loss_function.cc): rho = s, rho' = 1 for s <= 4; rho = 4 sqrt(s) - 4, rho' = 2/sqrt(s), rho'' < 0 beyond;
// Corrector (corrector.cc:88-111) with rho'' <= 0: residual and Jacobian are both scaled by sqrt(rho').
bool eval_line(const OptCam* cams, const int* res_cam, const OptObs* obs, long long r0, long long r1, const double x[4], double* cost,
               double g[4], double H[10])
{
    Jet4 line[4];
    for (int k = 0; k < 4; ++k) { line[k] = J(x[k]); line[k].v[k] = 1.0; }
    double c = 0.0;
    if (g) for (int k = 0; k < 4; ++k) g[k] = 0.0;
    if (H) for (int k = 0; k < 10; ++k) H[k] = 0.0;
    for (long long r = r0; r < r1; ++r) {
        Jet4 res[2];
        if (!reprojection_error(cams[res_cam[r]], obs[r], line, res)) return false;
        const double s = res[0].a * res[0].a + res[1].a * res[1].a;
        double rho, rho1;
        if (s > 4.0) { const double sr = std::sqrt(s); rho = 2.0 * 2.0 * sr - 4.0; rho1 = std::max(std::numeric_limits<double>::min(), 2.0 / sr); }
        else { rho = s; rho1 = 1.0; }
        c += 0.5 * rho;
        if (g) {
            const double w = std::sqrt(rho1);
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

// (A + diag(D2)) y = b for symmetric 4x4 A (upper triangle, row-wise: 00 01 02 03 11 12 13 22 23 33), Cholesky
bool solve4(const double A[10], const double D2[4], const double b[4], double y[4])
{
    double M[4][4];
    int idx = 0;
    for (int a = 0; a < 4; ++a) for (int c = a; c < 4; ++c) { M[a][c] = M[c][a] = A[idx++]; }
    for (int a = 0; a < 4; ++a) M[a][a] += D2[a];
    double L[4][4] = {{0}};
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j <= i; ++j) {
            double s = M[i][j];
            for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
            if (i == j) { if (!(s > 0.0)) return false; L[i][i] = std::sqrt(s); } else L[i][j] = s / L[j][j];
        }
    double z[4];
    for (int i = 0; i < 4; ++i) { double s = b[i]; for (int k = 0; k < i; ++k) s -= L[i][k] * z[k]; z[i] = s / L[i][i]; }
    for (int i = 3; i >= 0; --i) { double s = z[i]; for (int k = i + 1; k < 4; ++k) s -= L[k][i] * y[k]; y[i] = s / L[i][i]; }
    for (int i = 0; i < 4; ++i) if (!std::isfinite(y[i])) return false;
    return true;
}

// Pluecker -> Cayley (optimization.cc:34-91).  false: "symmetric line coords... do not bundle" (kept constant)
bool cayley_from_segment(const double* p, double x[4])
{
    V3 P1 = V(p[0], p[1], p[2]), P2 = V(p[3], p[4], p[5]);
    V3 l = normalized(P2 - P1);
    V3 m = crossd((P1 + P2) * 0.5, l);
    V3 e1, e2;
    if (normd(m) < L3D_EPS) {
        // the reference takes Eigen's FullPivLU kernel of l' here (a line through the origin of the translated frame, a set
        // of measure zero); any basis of the plane normal to l spans the same family of Cayley rotations
        V3 t = std::fabs(l.x) < 0.9 ? V(1, 0, 0) : V(0, 1, 0);
        e1 = normalized(crossd(l, t)); e2 = crossd(l, e1);
    } else { e1 = normalized(m); e2 = normalized(crossd(l, m)); }
    M3 Q, Qm, Qp;
    Q(0, 0) = l.x; Q(0, 1) = e1.x; Q(0, 2) = e2.x; Q(1, 0) = l.y; Q(1, 1) = e1.y; Q(1, 2) = e2.y; Q(2, 0) = l.z; Q(2, 1) = e1.z; Q(2, 2) = e2.z;
    for (int i = 0; i < 9; ++i) { Qm.m[i] = Q.m[i]; Qp.m[i] = Q.m[i]; }
    for (int i = 0; i < 3; ++i) { Qm(i, i) -= 1.0; Qp(i, i) += 1.0; }
    M3 sx = mul(Qm, inverse(Qp));
    x[0] = normd(m); x[1] = sx(2, 1); x[2] = sx(0, 2); x[3] = sx(1, 0);
    return !(std::isnan(x[0]) || std::isnan(x[1]) || std::isnan(x[2]) || std::isnan(x[3]));
}

// Cayley -> end points (optimization.cc:213-291); false if the new segment has no length (cluster dropped, 293-298)
bool segment_from_cayley(const double x[4], const double* old, double* out)
{
    V3 P1o = V(old[0], old[1], old[2]), P2o = V(old[3], old[4], old[5]), P1 = P1o, P2 = P2o;
    const double omega = x[0];
    if (!(omega < 0.0 || std::fabs(omega) < L3D_EPS)) {
        const double s0 = x[1], s1 = x[2], s2 = x[3], nm = s0 * s0 + s1 * s1 + s2 * s2, f = 1.0 / (1.0 + nm);
        // Q = f * ((1-nm) I + 2 [s]x + 2 s s')
        double Q[3][3] = {{(1.0 - nm) + 2.0 * s0 * s0, 2.0 * -s2 + 2.0 * s0 * s1, 2.0 * s1 + 2.0 * s0 * s2},
                          {2.0 * s2 + 2.0 * s1 * s0, (1.0 - nm) + 2.0 * s1 * s1, 2.0 * -s0 + 2.0 * s1 * s2},
                          {2.0 * -s1 + 2.0 * s2 * s0, 2.0 * s0 + 2.0 * s2 * s1, (1.0 - nm) + 2.0 * s2 * s2}};
        V3 l = V(f * Q[0][0], f * Q[1][0], f * Q[2][0]), m = V(f * Q[0][1], f * Q[1][1], f * Q[2][1]) * omega;
        if (std::fabs(l.x) > L3D_EPS || std::fabs(l.y) > L3D_EPS || std::fabs(l.z) > L3D_EPS) {
            V3 Pm = (P1o + P2o) * 0.5;
            double x1, x2, x3;
            if (std::fabs(l.x) > std::fabs(l.y) && std::fabs(l.x) > std::fabs(l.z)) { x1 = Pm.x; x3 = (-m.y - x1 * l.z) / -l.x; x2 = (m.z - x1 * l.y) / -l.x; }
            else if (std::fabs(l.y) > std::fabs(l.x) && std::fabs(l.y) > std::fabs(l.z)) { x2 = Pm.y; x3 = (m.x - x2 * l.z) / -l.y; x1 = (m.z + x2 * l.x) / l.y; }
            else { x3 = Pm.z; x2 = (m.x + x3 * l.y) / l.z; x1 = (-m.y + x3 * l.x) / l.z; }
            Pm = V(x1, x2, x3);
            P1 = Pm + l; P2 = Pm - l;
        }
    }
    out[0] = P1.x; out[1] = P1.y; out[2] = P1.z; out[3] = P2.x; out[4] = P2.y; out[5] = P2.z;
    return normd(P1 - P2) > L3D_EPS;
}

} // namespace

extern "C" {

// LineOptimizer::optimize.  cams: 16 doubles per camera (R row-major, C, fx, fy, px, py); res_xy: x1 y1 x2 y2 per residual
// (the float segment coordinates, optimization.cc:155-157); res_ptr[num_lines+1].  p1p2_out / valid_out per line
// (valid 0 = the cluster is dropped, optimization.cc:293-298).  summary (optional, 8 doubles): iterations, initial cost,
// final cost, termination (0 convergence, 1 no convergence, 2 failure), successful steps, free lines, final radius, 0.
int orc_optimize_lines(int num_lines, const double* p1p2, const long long* res_ptr, const int* res_cam, const double* res_xy, int num_cams,
                       const double* cams, int max_iter, double* p1p2_out, int* valid_out, double* summary)
{
    const int L = num_lines;
    std::vector<OptCam> C(num_cams);
    for (int i = 0; i < num_cams; ++i) {
        for (int k = 0; k < 9; ++k) C[i].R[k] = cams[16 * i + k];
        for (int k = 0; k < 3; ++k) C[i].C[k] = cams[16 * i + 9 + k];
        C[i].fx = cams[16 * i + 12]; C[i].fy = cams[16 * i + 13]; C[i].px = cams[16 * i + 14]; C[i].py = cams[16 * i + 15];
    }
    const long long NR = res_ptr[L];
    std::vector<OptObs> obs((size_t)NR);
    for (long long r = 0; r < NR; ++r) {
        OptObs& o = obs[(size_t)r];
        o.x1 = res_xy[4 * r]; o.y1 = res_xy[4 * r + 1]; o.x2 = res_xy[4 * r + 2]; o.y2 = res_xy[4 * r + 3];
        double dx = o.x2 - o.x1, dy = o.y2 - o.y1; const double n2 = dx * dx + dy * dy;
        if (n2 > 0) { const double n = std::sqrt(n2); dx /= n; dy /= n; }       // Eigen normalized()
        o.nx = -dy; o.ny = dx;
    }
    std::vector<double> x(4 * (size_t)L), xc(4 * (size_t)L), g(4 * (size_t)L), H(10 * (size_t)L), S(4 * (size_t)L, 1.0), diag(4 * (size_t)L), step(4 * (size_t)L);
    std::vector<char> free_(L);
    int nfree = 0;
    for (int i = 0; i < L; ++i) {
        free_[i] = cayley_from_segment(p1p2 + 6 * i, &x[4 * i]) && res_ptr[i + 1] > res_ptr[i];
        if (!free_[i] && !(res_ptr[i + 1] > res_ptr[i])) { /* no residuals: parameter block unused */ }
        else if (!free_[i]) { x[4 * i] = -1; x[4 * i + 1] = x[4 * i + 2] = x[4 * i + 3] = 0; }
        nfree += free_[i];
    }
    double sum[8] = {0, 0, 0, 1, 0, (double)nfree, 1e4, 0};
    auto finish = [&](int term, int iters, double c0, double c1, int nsucc, double radius) {
        for (int i = 0; i < L; ++i) valid_out[i] = segment_from_cayley(&x[4 * i], p1p2 + 6 * i, p1p2_out + 6 * i) ? 1 : 0;
        if (summary) { sum[0] = iters; sum[1] = c0; sum[2] = c1; sum[3] = term; sum[4] = nsucc; sum[5] = nfree; sum[6] = radius; for (int k = 0; k < 8; ++k) summary[k] = sum[k]; }
        return 0;
    };
    if (nfree == 0 || max_iter < 0) return finish(0, 0, 0, 0, 0, 1e4);
    // ---- iteration zero (trust_region_minimizer.cc: IterationZero)
    auto evaluate = [&](const std::vector<double>& xx, bool jac, double* total) {
        double c = 0.0; bool ok = true;
        for (int i = 0; i < L; ++i) {
            if (!free_[i]) continue;
            double ci;
            if (!eval_line(C.data(), res_cam, obs.data(), res_ptr[i], res_ptr[i + 1], &xx[4 * i], &ci, jac ? &g[4 * i] : nullptr, jac ? &H[10 * i] : nullptr)) { ok = false; continue; }
            c += ci;
        }
        *total = c; return ok;
    };
    double cost;
    if (!evaluate(x, true, &cost)) return finish(2, 0, 0, 0, 0, 1e4);
    const double cost0 = cost;
    static const int DI[4] = {0, 4, 7, 9};
    for (int i = 0; i < L; ++i) if (free_[i]) for (int k = 0; k < 4; ++k) S[4 * i + k] = 1.0 / (1.0 + std::sqrt(H[10 * i + DI[k]]));   // jacobi scaling
    auto grad_max = [&]() { double m = 0; for (int i = 0; i < L; ++i) if (free_[i]) for (int k = 0; k < 4; ++k) m = std::max(m, std::fabs(g[4 * i + k])); return m; };
    if (grad_max() <= 1e-10) return finish(0, 0, cost0, cost, 0, 1e4);
    double radius = 1e4, decrease_factor = 2.0; bool reuse_diagonal = false; int invalid = 0, nsucc = 0;
    int it = 0;
    for (;;) {
        if (it >= max_iter) return finish(1, it, cost0, cost, nsucc, radius);
        if (radius <= 1e-32) return finish(0, it, cost0, cost, nsucc, radius);
        ++it;
        // ---- LevenbergMarquardtStrategy::ComputeStep on the scaled system
        bool solved = true; double model_change = 0.0, step_sq = 0.0, x_sq = 0.0;
        for (int i = 0; i < L; ++i) {
            if (!free_[i]) continue;
            double Hs[10], gs[4], D2[4], y[4];
            int idx = 0;
            for (int a = 0; a < 4; ++a) { gs[a] = S[4 * i + a] * g[4 * i + a]; for (int b = a; b < 4; ++b) { Hs[idx] = S[4 * i + a] * S[4 * i + b] * H[10 * i + idx]; ++idx; } }
            if (!reuse_diagonal) for (int k = 0; k < 4; ++k) diag[4 * i + k] = std::min(std::max(Hs[DI[k]], 1e-6), 1e32);
            for (int k = 0; k < 4; ++k) D2[k] = diag[4 * i + k] / radius;
            if (!solve4(Hs, D2, gs, y)) { solved = false; continue; }
            double d[4], Hd[4] = {0, 0, 0, 0};
            for (int k = 0; k < 4; ++k) d[k] = -y[k];
            double Hf[4][4]; idx = 0;
            for (int a = 0; a < 4; ++a) for (int b = a; b < 4; ++b) { Hf[a][b] = Hf[b][a] = Hs[idx++]; }
            for (int a = 0; a < 4; ++a) for (int b = 0; b < 4; ++b) Hd[a] += Hf[a][b] * d[b];
            double dg = 0, dHd = 0;
            for (int k = 0; k < 4; ++k) { dg += d[k] * gs[k]; dHd += d[k] * Hd[k]; }
            model_change += -(dg + 0.5 * dHd);            // -(J d)'(r + J d / 2)
            for (int k = 0; k < 4; ++k) {
                step[4 * i + k] = d[k] * S[4 * i + k];
                xc[4 * i + k] = x[4 * i + k] + step[4 * i + k];
                step_sq += step[4 * i + k] * step[4 * i + k]; x_sq += x[4 * i + k] * x[4 * i + k];
            }
        }
        reuse_diagonal = true;
        if (!solved || !(model_change > 0.0)) {            // HandleInvalidStep
            if (++invalid >= 5) return finish(2, it, cost0, cost, nsucc, radius);
            radius *= 0.5; reuse_diagonal = false;
            continue;
        }
        invalid = 0;
        double cand;
        if (!evaluate(xc, false, &cand)) cand = std::numeric_limits<double>::max();
        if (std::sqrt(step_sq) <= 1e-8 * (std::sqrt(x_sq) + 1e-8)) return finish(0, it, cost0, cost, nsucc, radius);      // parameter tolerance
        if (std::fabs(cost - cand) <= 1e-6 * cost) return finish(0, it, cost0, cost, nsucc, radius);                     // function tolerance (the
                                                                                                   // candidate is NOT applied: both checks precede the acceptance test)
        const double quality = (cost - cand) / model_change;
        if (quality > 1e-3) {                                 // HandleSuccessfulStep
            for (int i = 0; i < L; ++i) if (free_[i]) for (int k = 0; k < 4; ++k) x[4 * i + k] = xc[4 * i + k];
            ++nsucc;
            if (!evaluate(x, true, &cost)) return finish(2, it, cost0, cost, nsucc, radius);
            radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * quality - 1.0, 3));
            radius = std::min(1e16, radius); decrease_factor = 2.0; reuse_diagonal = false;
            if (grad_max() <= 1e-10) return finish(0, it, cost0, cost, nsucc, radius);
        } else {                                              // HandleUnsuccessfulStep
            radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true;
        }
    }
}

}  // extern "C"

// ================================================================================================ pipeline
struct FinalLine {
    std::list<Seg3D> collinear;       // FinalLine3D::collinear3Dsegments_
    Seg3D cluster_seg;                // underlyingCluster_.seg3D_
    std::list<Seg2D> residuals;       // underlyingCluster_.residuals_
    uint32_t reference_view;
};

struct orc_ctx {
    bool by_wps, use_gpu;
    match_lines_fn_t match_fn; score_matches_fn_t score_fn; rdd_fn_t rdd_fn; collinear_fn_t collin_fn;
    orc_match_source_fn match_source;     // set: hands over every pair's match lists in place of matching, in both semantics
    std::map<uint32_t, View*> views; std::vector<uint32_t> view_order;
    std::map<uint32_t, std::vector<std::list<orc_match_t> > > matches;
    std::map<uint32_t, std::vector<orc_match_t> > scored;    // dump: flattened matches right after scoring
    std::map<uint32_t, unsigned> num_matches; std::map<uint32_t, bool> processed;
    std::map<uint32_t, std::set<uint32_t> > visual_neighbors, matched;
    std::map<uint32_t, std::list<uint32_t> > fixed_neighbors, views2wps; std::map<uint32_t, std::list<uint32_t> > wps2views;
    std::map<uint32_t, unsigned> num_wps; std::vector<float> views_avg_depths;
    std::map<uint32_t, std::map<uint32_t, M3> > fundamentals;
    std::vector<std::pair<Seg3D, orc_match_t> > est; std::map<Seg2D, size_t> entry_map;
    std::vector<std::pair<uint32_t, uint32_t> > pairs; long long pair_evals;
    // params
    unsigned num_neighbors, visibility_t; float sigma_p, sigma_a, two_sigA_sqr, epi, const_reg_depth, med_scene_depth, med_scene_depth_lines, collin_t;
    int kNN; bool fixed3Dreg, perform_RDD; size_t num_lines_total;
    V3 translation;
    // affinity
    std::list<CLEdge> A, A_raw, A_final; std::map<Seg2D, int> global2local; std::map<int, Seg2D> local2global; std::vector<Seg2D> l2g_dump; int localID;
    std::map<Seg2D, std::set<Seg2D> > used;
    std::vector<FinalLine> clusters3D, lines3D;
    double opt_summary[8];
};

namespace {

void perform_translation(orc_ctx* c, V3 t)   // line3D.cc:548-575
{
    for (size_t i = 0; i < c->view_order.size(); ++i) c->views[c->view_order[i]]->translate(t);
    for (size_t i = 0; i < c->lines3D.size(); ++i) {
        for (std::list<Seg3D>::iterator it = c->lines3D[i].collinear.begin(); it != c->lines3D[i].collinear.end(); ++it) it->translate(t);
        c->lines3D[i].cluster_seg.translate(t);
    }
}
void translate(orc_ctx* c)                   // line3D.cc:500-536
{
    if (c->views.empty()) return;
    double tr[3] = {0, 0, 0};
    for (int i = 0; i < 3; ++i) {
        std::vector<double> coords;
        for (std::map<uint32_t, View*>::const_iterator it = c->views.begin(); it != c->views.end(); ++it) {
            double val = i == 0 ? it->second->C.x : (i == 1 ? it->second->C.y : it->second->C.z);
            if (std::fabs(val) > L3D_EPS) coords.push_back(val);
        }
        if (!coords.empty()) { std::sort(coords.begin(), coords.end()); tr[i] = coords[coords.size() / 2]; }
    }
    c->translation = V(tr[0], tr[1], tr[2]);
    perform_translation(c, c->translation * -1.0);
}
void untranslate(orc_ctx* c) { perform_translation(c, c->translation); }   // line3D.cc:539-545

Seg3D unproject_match(orc_ctx* c, const orc_match_t& m, bool src = true)   // line3D.cc:1556-1568
{
    if (src) return c->views[m.src_cam]->unprojectSegment(m.src_seg, m.d_p1, m.d_p2);
    return c->views[m.tgt_cam]->unprojectSegment(m.tgt_seg, m.d_q1, m.d_q2);
}

void find_visual_neighbors_from_wps(orc_ctx* c, uint32_t camID)   // line3D.cc:578-699
{
    c->visual_neighbors[camID].clear();
    std::map<uint32_t, unsigned> common;
    for (std::list<uint32_t>::const_iterator w = c->views2wps[camID].begin(); w != c->views2wps[camID].end(); ++w)
        for (std::list<uint32_t>::const_iterator v = c->wps2views[*w].begin(); v != c->wps2views[*w].end(); ++v)
            if (*v != camID) ++common[*v];
    if (common.empty()) return;
    struct VN { uint32_t cam; float score, axisAngle, dist; };
    std::list<VN> nb; View* v = c->views[camID];
    for (std::map<uint32_t, unsigned>::const_iterator it = common.begin(); it != common.end(); ++it) {
        VN vn; vn.cam = it->first;
        vn.score = 2.0f * float(it->second) / float(c->num_wps[camID] + c->num_wps[it->first]);
        vn.axisAngle = (float)v->opticalAxesAngle(*c->views[it->first]);
        vn.dist = v->distanceVisualNeighborScore(*c->views[it->first]);
        if (vn.axisAngle < 1.571f && it->second > 4) nb.push_back(vn);
    }
    nb.sort([](const VN& a, const VN& b) { return a.score > b.score; });
    if (nb.size() > c->num_neighbors) {
        std::list<VN> tmp = nb;
        float score_t = 0.80f * nb.front().score; unsigned nbig = 0;
        for (std::list<VN>::const_iterator n = nb.begin(); n != nb.end() && n->score > score_t; ++n) ++nbig;
        nb.resize(nbig);
        nb.sort([](const VN& a, const VN& b) { return a.dist > b.dist; });
        if (nb.size() > c->num_neighbors / 2) nb.resize(c->num_neighbors / 2);
        nb.splice(nb.end(), tmp);
    }
    std::set<uint32_t> usedn; float min_baseline = 0.1f;
    for (std::list<VN>::const_iterator n = nb.begin(); n != nb.end() && usedn.size() < c->num_neighbors; ++n) {
        View* v2 = c->views[n->cam];
        if (usedn.find(n->cam) == usedn.end() && v->baseLine(*v2) > min_baseline) {
            bool valid = true;
            for (std::set<uint32_t>::const_iterator u = usedn.begin(); u != usedn.end() && valid; ++u)
                if (!(v->baseLine(*c->views[*u]) > min_baseline)) valid = false;
            if (valid) usedn.insert(n->cam);
        }
    }
    c->visual_neighbors[camID] = usedn;
}

M3 fundamental(orc_ctx* c, View* src, View* tgt)   // line3D.cc:861-897
{
    if (c->fundamentals[src->id].count(tgt->id)) return c->fundamentals[src->id][tgt->id];
    if (c->fundamentals[tgt->id].count(src->id)) return transpose(c->fundamentals[tgt->id][src->id]);
    M3 R = mul(tgt->R, transpose(src->R));
    V3 t = tgt->t - mul(R, src->t);
    M3 T; T(0, 0) = 0; T(0, 1) = -t.z; T(0, 2) = t.y; T(1, 0) = t.z; T(1, 1) = 0; T(1, 2) = -t.x; T(2, 0) = -t.y; T(2, 1) = t.x; T(2, 2) = 0;
    M3 E = mul(T, R);
    M3 F = mul(mul(inverse(transpose(tgt->K)), E), inverse(src->K));
    c->fundamentals[src->id][tgt->id] = F;
    return F;
}

void matching(orc_ctx* c, uint32_t src, uint32_t tgt, const M3& F)   // matchingGPU 1040-1074 / matchingCPU 900-1015
{
    View* v1 = c->views[src]; View* v2 = c->views[tgt];
    int Ns = (int)v1->lines.size(), Nt = (int)v2->lines.size();
    int cap = c->kNN > 0 ? c->kNN : Nt;
    std::vector<int> counts(Ns); std::vector<orc_match_t> out((size_t)Ns * cap);
    long long n;
    if (c->match_source) {
        n = c->match_source(src, tgt, Ns, Nt, c->kNN, &counts[0], &out[0], cap);
    } else if (c->use_gpu) {
        float Ff[9]; for (int i = 0; i < 9; ++i) Ff[i] = (float)F.m[i];   // eigen2dataArray line3D.cc:2775-2781
        n = c->match_fn(&v1->lines[0].x, Ns, &v2->lines[0].x, Nt, Ff, v1->RtKinv_f, v2->RtKinv_f, v1->C_f3, v2->C_f3,
                        src, tgt, c->epi, c->kNN, &counts[0], &out[0], cap, NULL);
    } else {
        double C1[3] = {v1->C.x, v1->C.y, v1->C.z}, C2[3] = {v2->C.x, v2->C.y, v2->C.z};
        n = orc_match_lines_f64(&v1->lines[0].x, Ns, &v2->lines[0].x, Nt, F.m, v1->RtKinv.m, v2->RtKinv.m, C1, C2,
                                src, tgt, c->epi, c->kNN, &counts[0], &out[0], cap, NULL);
    }
    for (int r = 0; r < Ns; ++r)
        for (int i = 0; i < counts[r] && i < cap; ++i) c->matches[src][r].push_back(out[(size_t)r * cap + i]);
    c->num_matches[src] += (unsigned)n;
    c->pairs.push_back(std::make_pair(src, tgt));
    c->pair_evals += (long long)Ns * Nt;
}

void check_match_orientation(orc_ctx* c, uint32_t src)   // line3D.cc:811-858
{
    unsigned num = 0;
    std::vector<std::list<orc_match_t> >& M = c->matches[src];
    for (size_t i = 0; i < M.size(); ++i) {
        std::list<orc_match_t> remaining;
        for (std::list<orc_match_t>::const_iterator it = M[i].begin(); it != M[i].end(); ++it) {
            Seg3D s = unproject_match(c, *it);
            double ang = c->views[it->src_cam]->segmentQualityAngle(s, it->src_seg);
            if (ang > L3D_PI_1_32 && ang < L3D_PI_31_32) remaining.push_back(*it);
        }
        M[i] = remaining; num += (unsigned)remaining.size();
    }
    c->num_matches[src] = num;
}

bool sort_by_ids(const orc_match_t& a, const orc_match_t& b)   // commons.h:206-214
{ return a.tgt_cam < b.tgt_cam || (a.tgt_cam == b.tgt_cam && a.tgt_seg < b.tgt_seg); }

void scoring_gpu(orc_ctx* c, uint32_t src)   // line3D.cc:1297-1414
{
    View* v = c->views[src];
    if (c->num_matches[src] == 0) return;
    std::vector<std::list<orc_match_t> >& M = c->matches[src];
    for (size_t i = 0; i < M.size(); ++i) M[i].sort(sort_by_ids);
    size_t N = v->lines.size();
    std::vector<int> ranges(2 * N); unsigned offset = 0;
    for (size_t i = 0; i < N; ++i) {
        if (!M[i].empty()) { ranges[2 * i] = (int)offset; ranges[2 * i + 1] = (int)(offset + M[i].size() - 1); offset += (unsigned)M[i].size(); }
        else { ranges[2 * i] = -1; ranges[2 * i + 1] = -1; }
    }
    unsigned nm = c->num_matches[src];
    std::vector<float> mat(4 * (size_t)nm), reg(2 * (size_t)nm), scores(nm);
    for (size_t i = 0; i < M.size(); ++i) {
        int off = ranges[2 * i]; if (off < 0) continue;
        int id = 0;
        for (std::list<orc_match_t>::const_iterator it = M[i].begin(); it != M[i].end(); ++it, ++id) {
            float* m = &mat[4 * (size_t)(off + id)];
            m[0] = (float)i; m[1] = (float)it->tgt_cam; m[2] = it->d_p1; m[3] = it->d_p2;
            Seg3D s = v->unprojectSegment(it->src_seg, it->d_p1, it->d_p2);
            reg[2 * (size_t)(off + id)] = c->views[it->tgt_cam]->regularizerFrom3Dpoint(s.P1);
            reg[2 * (size_t)(off + id) + 1] = c->views[it->tgt_cam]->regularizerFrom3Dpoint(s.P2);
        }
    }
    c->score_fn(&v->lines[0].x, (int)N, &mat[0], (int)nm, &ranges[0], &reg[0], v->RtKinv_f, v->C_f3, c->two_sigA_sqr, v->k,
                MIN_SIMILARITY_3D, &scores[0], NULL);
    for (size_t i = 0; i < M.size(); ++i) {
        int off = ranges[2 * i]; if (off < 0) continue;
        int id = 0;
        for (std::list<orc_match_t>::iterator it = M[i].begin(); it != M[i].end(); ++it, ++id) it->score3D = scores[off + id];
    }
}

float angle_between_seg3d(const Seg3D& s1, const Seg3D& s2)   // line3D.cc:1571-1583 (undirected)
{
    float dot_p = (float)dotd(s1.dir, s2.dir);
    float angle = (float)((double)acosf(fmaxf(fminf(dot_p, 1.0f), -1.0f)) / PI_D * (double)180.0f);
    if (angle > 90.0f) angle = 180.0f - angle;
    return angle;
}

void scoring_cpu(orc_ctx* c, uint32_t src)   // line3D.cc:1208-1294 + similarityForScoring 1417-1446
{
    View* v = c->views[src]; float k = v->k;
    std::vector<std::list<orc_match_t> >& Mv = c->matches[src];
    for (size_t i = 0; i < Mv.size(); ++i)
        for (std::list<orc_match_t>::iterator it = Mv[i].begin(); it != Mv[i].end(); ++it) {
            orc_match_t M = *it; float score3D = 0.0f; std::map<uint32_t, float> per_cam;
            Seg3D M3D = v->unprojectSegment(M.src_seg, M.d_p1, M.d_p2);
            float sig1 = M.d_p1 * k, sig2 = M.d_p2 * k;
            float reg1 = 2.0f * sig1 * sig1, reg2 = 2.0f * sig2 * sig2;
            float s1t = c->views[M.tgt_cam]->regularizerFrom3Dpoint(M3D.P1), s2t = c->views[M.tgt_cam]->regularizerFrom3Dpoint(M3D.P2);
            reg1 = 0.5f * (reg1 + 2.0f * s1t * s1t); reg2 = 0.5f * (reg2 + 2.0f * s2t * s2t);
            for (std::list<orc_match_t>::const_iterator it2 = Mv[i].begin(); it2 != Mv[i].end(); ++it2) {
                const orc_match_t& M2 = *it2;
                if (M.tgt_cam == M2.tgt_cam) continue;
                float sim = 0.0f;
                Seg3D s2 = unproject_match(c, M2, true);
                if (!(M3D.length < L3D_EPS || s2.length < L3D_EPS)) {
                    float angle = angle_between_seg3d(M3D, s2);
                    float sim_a = expf(-angle * angle / c->two_sigA_sqr);
                    float sim_p = 0.0f;
                    if (M.src_cam == M2.src_cam && M.src_seg == M2.src_seg) {
                        float d1 = M.d_p1 - M2.d_p1, d2 = M.d_p2 - M2.d_p2;
                        sim_p = fminf(expf(-d1 * d1 / reg1), expf(-d2 * d2 / reg2));
                    }
                    float s = fminf(sim_a, sim_p);
                    sim = s > MIN_SIMILARITY_3D ? s : 0.0f;
                }
                std::map<uint32_t, float>::iterator pc = per_cam.find(M2.tgt_cam);
                if (pc != per_cam.end()) { if (sim > pc->second) { score3D -= pc->second; score3D += sim; pc->second = sim; } }
                else { score3D += sim; per_cam[M2.tgt_cam] = sim; }
            }
            it->score3D = score3D;
        }
}

void store_inverse_matches(orc_ctx* c, uint32_t src)   // line3D.cc:1672-1699
{
    std::vector<std::list<orc_match_t> >& M = c->matches[src];
    for (size_t i = 0; i < M.size(); ++i)
        for (std::list<orc_match_t>::const_iterator it = M[i].begin(); it != M[i].end(); ++it) {
            const orc_match_t& m = *it;
            if (m.score3D > 0.0f && !c->processed[m.tgt_cam]) {
                orc_match_t inv = m;
                inv.src_cam = m.tgt_cam; inv.src_seg = m.tgt_seg; inv.tgt_cam = m.src_cam; inv.tgt_seg = m.src_seg;
                inv.d_p1 = m.d_q1; inv.d_p2 = m.d_q2; inv.d_q1 = m.d_p1; inv.d_q2 = m.d_p2; inv.score3D = 0.0f;
                c->matches[m.tgt_cam][m.tgt_seg].push_back(inv);
                ++c->num_matches[m.tgt_cam];
            }
        }
}

void filter_matches(orc_ctx* c, uint32_t src)   // line3D.cc:1586-1669
{
    std::vector<float> depths; float max_score = 0.0f;
    std::vector<std::list<orc_match_t> >& M = c->matches[src];
    for (size_t i = 0; i < M.size(); ++i)
        for (std::list<orc_match_t>::const_iterator it = M[i].begin(); it != M[i].end(); ++it) max_score = fmaxf(max_score, it->score3D);
    float score_lim = MIN_BEST_SCORE_PERC * max_score;
    unsigned num_valid = 0;
    for (size_t i = 0; i < M.size(); ++i) {
        orc_match_t best; memset(&best, 0, sizeof(best)); best.score3D = 0.0f;
        std::list<orc_match_t> ms = M[i]; M[i].clear();
        for (std::list<orc_match_t>::const_iterator it = ms.begin(); it != ms.end(); ++it)
            if (it->score3D > 0.0f && it->score3D > score_lim) { M[i].push_back(*it); if (it->score3D > best.score3D) best = *it; }
        num_valid += (unsigned)M[i].size();
        if (best.score3D > MIN_BEST_SCORE_3D) {
            Seg2D seg = {src, (uint32_t)i};
            Seg3D s = unproject_match(c, best, true);
            c->entry_map[seg] = c->est.size();
            c->est.push_back(std::make_pair(s, best));
            depths.push_back(best.d_p1); depths.push_back(best.d_p2);
        } else M[i].clear();
    }
    c->num_matches[src] = num_valid;   // counted before rejected lists are cleared, like line3D.cc:1630-1655
    float med = (float)L3D_EPS;
    if (!depths.empty()) { std::sort(depths.begin(), depths.end()); med = depths[depths.size() / 2]; }
    if (!c->fixed3Dreg) c->views[src]->update_median_depth(med, -1.0f, c->med_scene_depth);
    else c->views[src]->update_median_depth(med, c->sigma_p, c->med_scene_depth);
}

void compute_matches(orc_ctx* c)   // line3D.cc:702-778
{
    for (std::map<uint32_t, std::set<uint32_t> >::const_iterator it = c->visual_neighbors.begin(); it != c->visual_neighbors.end(); ++it) {
        uint32_t src = it->first;
        for (std::set<uint32_t>::const_iterator n = it->second.begin(); n != it->second.end(); ++n)
            if (c->matched[src].find(*n) == c->matched[src].end()) {
                M3 F = fundamental(c, c->views[src], c->views[*n]);
                matching(c, src, *n, F);
                c->matched[src].insert(*n); c->matched[*n].insert(src);
            }
        check_match_orientation(c, src);                  // L3D_DEF_CHECK_MATCH_ORIENTATION true (commons.h:56)
        if (c->use_gpu) scoring_gpu(c, src); else scoring_cpu(c, src);
        {   // dump for stage-level parity tests
            std::vector<orc_match_t>& d = c->scored[src]; d.clear();
            for (size_t i = 0; i < c->matches[src].size(); ++i)
                for (std::list<orc_match_t>::const_iterator m = c->matches[src][i].begin(); m != c->matches[src][i].end(); ++m) d.push_back(*m);
        }
        store_inverse_matches(c, src);
        filter_matches(c, src);
        c->processed[src] = true;
    }
}

// similarity(s1,m1,seg2,truncate) (line3D.cc:1467-1553)
float similarity(orc_ctx* c, const Seg3D& s1, const orc_match_t& m1, const Seg2D& seg2, bool truncate)
{
    std::map<Seg2D, size_t>::const_iterator e2 = c->entry_map.find(seg2);
    if (e2 == c->entry_map.end()) return 0.0f;
    const Seg3D& s2 = c->est[e2->second].first; const orc_match_t& m2 = c->est[e2->second].second;
    if (s1.length < L3D_EPS || s2.length < L3D_EPS) return 0.0f;
    View* v1 = c->views[m1.src_cam]; View* v2 = c->views[m2.src_cam];
    float angle = angle_between_seg3d(s1, s2);
    float sim_a = expf(-angle * angle / c->two_sigA_sqr);
    float cutoff1 = v1->median_depth, cutoff2 = v2->median_depth;
    if (c->med_scene_depth_lines > L3D_EPS) { cutoff1 = fminf(cutoff1, c->med_scene_depth_lines); cutoff2 = fminf(cutoff2, c->med_scene_depth_lines); }
    float d11 = s2.distance_Point2Line(s1.P1), d12 = s2.distance_Point2Line(s1.P2);
    float d21 = s1.distance_Point2Line(s2.P1), d22 = s1.distance_Point2Line(s2.P2);
    float sig11 = m1.d_p1 > cutoff1 ? cutoff1 * v1->k : m1.d_p1 * v1->k;
    float sig12 = m1.d_p2 > cutoff1 ? cutoff1 * v1->k : m1.d_p2 * v1->k;
    float reg11 = 2.0f * sig11 * sig11, reg12 = 2.0f * sig12 * sig12;
    float sig21 = m2.d_p1 > cutoff2 ? cutoff2 * v2->k : m2.d_p1 * v2->k;
    float sig22 = m2.d_p2 > cutoff2 ? cutoff2 * v2->k : m2.d_p2 * v2->k;
    float reg21 = 2.0f * sig21 * sig21, reg22 = 2.0f * sig22 * sig22;
    float sim_p1 = fminf(expf(-d11 * d11 / reg11), expf(-d12 * d12 / reg12));
    float sim_p2 = fminf(expf(-d21 * d21 / reg21), expf(-d22 * d22 / reg22));
    float sim = fminf(sim_a, fminf(sim_p1, sim_p2));
    if (truncate) return sim > MIN_SIMILARITY_3D ? sim : 0.0f;
    return sim;
}

bool unused_pair(orc_ctx* c, const Seg2D& a, const Seg2D& b)   // line3D.cc:1982-2002
{
    if (c->used[a].find(b) != c->used[a].end()) return false;
    c->used[a].insert(b); c->used[b].insert(a);
    return true;
}
int local_id(orc_ctx* c, const Seg2D& s)   // line3D.cc:2005-2023
{
    std::map<Seg2D, int>::const_iterator it = c->global2local.find(s);
    if (it != c->global2local.end()) return it->second;
    int id = c->localID++;
    c->global2local[s] = id; c->local2global[id] = s;
    return id;
}

// View::findCollinearSegments (view.cc:152-171) -> findCollinGPU (173-209: dense char matrix from the kernel, scanned per
// row in ascending column order) or findCollinCPU (212-263)
void view_find_collinear(orc_ctx* c, View* v, float dist_t, bool useGPU)
{
    if (std::fabs(dist_t - v->collin_t) < L3D_EPS) return;      // already computed
    if (!(dist_t > L3D_EPS)) return;
    v->collin_t = dist_t;
    const int N = (int)v->lines.size();
    v->collin.assign(N, std::list<uint32_t>());
    if (N == 0) return;
    std::vector<unsigned char> C((size_t)N * N);
    if (useGPU) c->collin_fn((const float*)v->lines.data(), N, dist_t, C.data(), nullptr);
    else orc_collinear_f64((const float*)v->lines.data(), N, dist_t, C.data(), nullptr);
    for (int i = 0; i < N; ++i)
        for (int x = 0; x < N; ++x)
            if (C[(size_t)i * N + x] == 1) v->collin[i].push_back((uint32_t)x);
}
std::list<uint32_t> collinear_segments(View* v, uint32_t seg)   // View::collinearSegments view.cc:281-287
{
    if (v->collin.size() == v->lines.size() && seg < v->lines.size()) return v->collin[seg];
    return std::list<uint32_t>();
}

void computing_affinity_matrix(orc_ctx* c)   // line3D.cc:1852-1979
{
    c->A.clear(); c->global2local.clear(); c->local2global.clear(); c->localID = 0; c->used.clear();
    const bool collin = c->collin_t > L3D_EPS;
    for (size_t i = 0; i < c->est.size(); ++i) {
        const Seg3D& s = c->est[i].first; const orc_match_t& m = c->est[i].second;
        Seg2D seg = {m.src_cam, m.src_seg}; int id1 = -1; bool found_aff = false;
        const std::list<orc_match_t>& L = c->matches[m.src_cam][m.src_seg];
        for (std::list<orc_match_t>::const_iterator it = L.begin(); it != L.end(); ++it) {
            Seg2D seg2 = {it->tgt_cam, it->tgt_seg};
            float sim = similarity(c, s, m, seg2, false);
            if (sim > MIN_AFFINITY && unused_pair(c, seg, seg2)) {
                if (id1 < 0) id1 = local_id(c, seg);
                int id2 = local_id(c, seg2);
                CLEdge e = {id1, id2, sim}; c->A.push_back(e);
                CLEdge e2 = {id2, id1, sim}; c->A.push_back(e2);
                found_aff = true;
                if (collin) {            // links to the segments collinear with the target (line3D.cc:1904-1937)
                    std::list<uint32_t> coll = collinear_segments(c->views[seg2.cam], seg2.seg);
                    for (std::list<uint32_t>::const_iterator cit = coll.begin(); cit != coll.end(); ++cit) {
                        Seg2D sc = {seg2.cam, *cit};
                        float simc = similarity(c, s, m, sc, false);
                        if (simc > MIN_AFFINITY && unused_pair(c, seg, sc)) {
                            int idc = local_id(c, sc);
                            CLEdge a = {id1, idc, simc}; c->A.push_back(a);
                            CLEdge b = {idc, id1, simc}; c->A.push_back(b);
                        }
                    }
                }
            }
        }
        if (found_aff && id1 >= 0 && collin) {   // links to the segments collinear with the source (line3D.cc:1941-1974)
            std::list<uint32_t> coll = collinear_segments(c->views[seg.cam], seg.seg);
            for (std::list<uint32_t>::const_iterator cit = coll.begin(); cit != coll.end(); ++cit) {
                Seg2D sc = {seg.cam, *cit};
                float simc = similarity(c, s, m, sc, false);
                if (simc > MIN_AFFINITY && unused_pair(c, seg, sc)) {
                    int idc = local_id(c, sc);
                    CLEdge a = {id1, idc, simc}; c->A.push_back(a);
                    CLEdge b = {idc, id1, simc}; c->A.push_back(b);
                }
            }
        }
    }
    c->used.clear();
}

void perform_rdd(orc_ctx* c)   // line3D.cc:2026-2076
{
    int n = (int)c->global2local.size(); int ne = (int)c->A.size();
    std::vector<int> ei(ne), ej(ne), oi(ne), oj(ne); std::vector<float> ew(ne), ow(ne);
    int p = 0;
    for (std::list<CLEdge>::const_iterator it = c->A.begin(); it != c->A.end(); ++it, ++p) { ei[p] = it->i; ej[p] = it->j; ew[p] = it->w; }
    c->rdd_fn(ne, &ei[0], &ej[0], &ew[0], n, &oi[0], &oj[0], &ow[0], NULL);
    c->A.clear();
    std::map<int, std::map<int, float> > entries;
    for (int i = 0; i < ne; ++i) {
        int s1 = oi[i], s2 = oj[i]; float w12 = ow[i], w21 = w12;
        if (entries[s2].find(s1) != entries[s2].end()) w21 = entries[s2][s1];
        float w = fminf(w12, w21);
        entries[s1][s2] = w; entries[s2][s1] = w;
    }
    for (std::map<int, std::map<int, float> >::const_iterator it = entries.begin(); it != entries.end(); ++it)
        for (std::map<int, float>::const_iterator it2 = it->second.begin(); it2 != it->second.end(); ++it2) {
            CLEdge e = {it->first, it2->first, it2->second}; c->A.push_back(e);
        }
}

// symmetric 3x3 eigen-decomposition (cyclic Jacobi).  Stands in for Eigen::JacobiSVD of the PSD scatter matrix
// (line3D.cc:2196-2211): for a symmetric PSD matrix U's dominant column == dominant eigenvector (up to sign).
void dominant_eigenvector(double S[3][3], double out[3])
{
    double Vm[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 64; ++sweep) {
        double off = S[0][1] * S[0][1] + S[0][2] * S[0][2] + S[1][2] * S[1][2];
        if (off < 1e-300) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (std::fabs(S[p][q]) < 1e-300) continue;
                double theta = (S[q][q] - S[p][p]) / (2.0 * S[p][q]);
                double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                double cs = 1.0 / std::sqrt(t * t + 1.0), sn = t * cs;
                for (int k = 0; k < 3; ++k) { double a = S[k][p], b = S[k][q]; S[k][p] = cs * a - sn * b; S[k][q] = sn * a + cs * b; }
                for (int k = 0; k < 3; ++k) { double a = S[p][k], b = S[q][k]; S[p][k] = cs * a - sn * b; S[q][k] = sn * a + cs * b; }
                for (int k = 0; k < 3; ++k) { double a = Vm[k][p], b = Vm[k][q]; Vm[k][p] = cs * a - sn * b; Vm[k][q] = sn * a + cs * b; }
            }
    }
    int mx = 0; if (S[1][1] > S[mx][mx]) mx = 1; if (S[2][2] > S[mx][mx]) mx = 2;
    out[0] = Vm[0][mx]; out[1] = Vm[1][mx]; out[2] = Vm[2][mx];
}

bool line_from_cluster(orc_ctx* c, const std::list<Seg2D>& cluster, FinalLine& LC)   // get3DlineFromCluster line3D.cc:2155-2218
{
    V3 P = V(0, 0, 0); int n = (int)cluster.size() * 2;
    std::vector<V3> pts; uint32_t reference_cam = 0; float max_len_2D = 0.0f;
    for (std::list<Seg2D>::const_iterator it = cluster.begin(); it != cluster.end(); ++it) {
        const Seg3D& h = c->est[c->entry_map[*it]].first;
        P = P + h.P1; P = P + h.P2; pts.push_back(h.P1); pts.push_back(h.P2);
        f4 co = c->views[it->cam]->lines[it->seg];
        float l2 = (co.x - co.z) * (co.x - co.z) + (co.y - co.w) * (co.y - co.w);
        if (l2 > max_len_2D) { max_len_2D = l2; reference_cam = it->cam; }
    }
    P = V(P.x / double(n), P.y / double(n), P.z / double(n));
    double S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (size_t i = 0; i < pts.size(); ++i) {
        double d[3] = {pts[i].x - P.x, pts[i].y - P.y, pts[i].z - P.z};
        for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) S[a][b] += d[a] * d[b];
    }
    double dv[3]; dominant_eigenvector(S, dv);
    V3 dir = normalized(V(dv[0], dv[1], dv[2]));
    LC.cluster_seg = Seg3D(P - dir, P + dir); LC.residuals = cluster; LC.reference_view = reference_cam; LC.collinear.clear();
    return !cluster.empty();
}

void cluster_segments(orc_ctx* c)   // line3D.cc:2079-2152
{
    c->clusters3D.clear(); c->lines3D.clear();
    c->A_final = c->A;
    if (c->A.empty()) return;
    Universe* u = perform_clustering(c->A, (int)c->global2local.size(), 3.0f);
    c->A.clear();
    std::map<int, std::list<Seg2D> > cl2seg; std::map<int, std::map<uint32_t, bool> > cl2cam; std::vector<int> uniq;
    for (std::map<int, Seg2D>::const_iterator it = c->local2global.begin(); it != c->local2global.end(); ++it) {
        int cl = u->find(it->first);
        if (cl2seg.find(cl) == cl2seg.end()) uniq.push_back(cl);
        cl2seg[cl].push_back(it->second); cl2cam[cl][it->second.cam] = true;
    }
    delete u;
    for (size_t i = 0; i < uniq.size(); ++i)
        if (cl2cam[uniq[i]].size() >= c->visibility_t) {
            FinalLine LC;
            if (line_from_cluster(c, cl2seg[uniq[i]], LC)) c->clusters3D.push_back(LC);
        }
}

// project2DsegmentOnto3Dline (line3D.cc:2221-2266)
Seg3D project_onto_line(orc_ctx* c, const Seg2D& s2, const Seg3D& s3, bool& ok)
{
    V3 P = s3.P1, u = s3.dir; View* v = c->views[s2.cam]; V3 Q = v->C;
    f4 l = v->lines[s2.seg];
    V3 v1 = v->ray(V(l.x, l.y, 1.0)), v2 = v->ray(V(l.z, l.w, 1.0));   // getNormalizedLinePointRay view.cc:324-353
    V3 w = P - Q;
    double a = dotd(u, u), b1 = dotd(u, v1), b2 = dotd(u, v2), c1 = dotd(v1, v1), c2 = dotd(v2, v2), d = dotd(u, w), e1 = dotd(v1, w), e2 = dotd(v2, w);
    double den1 = a * c1 - b1 * b1, den2 = a * c2 - b2 * b2;
    if (std::fabs(den1) > L3D_EPS && std::fabs(den2) > L3D_EPS) {
        ok = true;
        double s1 = (b1 * e1 - c1 * d) / den1, s2_ = (b2 * e2 - c2 * d) / den2;
        return Seg3D(P + u * s1, P + u * s2_);
    }
    ok = false; return Seg3D();
}

std::list<Seg3D> find_collinear_segments(orc_ctx* c, const FinalLine& cl)   // line3D.cc:2342-2452
{
    std::list<Seg3D> out;
    V3 COG = (cl.cluster_seg.P1 + cl.cluster_seg.P2) * 0.5;
    struct LP { size_t lineID, pointID, camID; float dist; };
    std::list<LP> lp; std::vector<V3> pts(cl.residuals.size() * 2);
    float distToCOG = 0.0f; V3 border = V(0, 0, 0);
    size_t pID = 0, id = 0;
    for (std::list<Seg2D>::const_iterator it = cl.residuals.begin(); it != cl.residuals.end(); ++it, ++id, pID += 2) {
        bool ok; Seg3D proj = project_onto_line(c, *it, cl.cluster_seg, ok);
        if (!ok) continue;
        LP p1 = {id, pID, it->cam, 0.0f}; pts[pID] = proj.P1; lp.push_back(p1);
        float d = (float)normd(proj.P1 - COG); if (d > distToCOG) { distToCOG = d; border = proj.P1; }
        LP p2 = {id, pID + 1, it->cam, 0.0f}; pts[pID + 1] = proj.P2; lp.push_back(p2);
        d = (float)normd(proj.P2 - COG); if (d > distToCOG) { distToCOG = d; border = proj.P2; }
    }
    if (lp.size() < 6) return out;
    for (std::list<LP>::iterator l = lp.begin(); l != lp.end(); ++l) l->dist = (float)normd(pts[l->pointID] - border);
    lp.sort([](const LP& a, const LP& b) { return a.dist < b.dist; });
    std::map<size_t, unsigned> open; std::map<size_t, bool> open_lines; bool opened = false; V3 cur = V(0, 0, 0);
    for (std::list<LP>::const_iterator l = lp.begin(); l != lp.end(); ++l) {
        if (open_lines.find(l->lineID) == open_lines.end()) { open_lines[l->lineID] = true; ++open[l->camID]; }
        else { open_lines.erase(l->lineID); --open[l->camID]; if (open[l->camID] == 0) open.erase(l->camID); }
        if (opened && open.size() < 3) { out.push_back(Seg3D(cur, pts[l->pointID])); opened = false; }
        else if (!opened && open.size() >= 3) { cur = pts[l->pointID]; opened = true; }
    }
    return out;
}

} // namespace

extern "C" {

orc_ctx* orc_create(int neighbors_by_worldpoints, int use_gpu)
{
    orc_ctx* c = new orc_ctx();
    c->by_wps = neighbors_by_worldpoints != 0; c->use_gpu = use_gpu != 0;
    c->match_fn = (match_lines_fn_t)orc_match_lines_f32; c->score_fn = (score_matches_fn_t)orc_score_matches_f32; c->rdd_fn = (rdd_fn_t)orc_rdd_f32;
    c->collin_fn = (collinear_fn_t)orc_collinear_f32; c->match_source = NULL;
    c->num_lines_total = 0; c->pair_evals = 0; c->collin_t = -1.0f; c->localID = 0;
    c->translation = V(0, 0, 0); c->med_scene_depth = -1.0f; c->med_scene_depth_lines = 0.0f;
    c->fixed3Dreg = false; c->perform_RDD = false; c->visibility_t = 3; c->num_neighbors = 10; c->kNN = 10;
    return c;
}
void orc_destroy(orc_ctx* c)
{
    if (!c) return;
    for (std::map<uint32_t, View*>::iterator it = c->views.begin(); it != c->views.end(); ++it) delete it->second;
    delete c;
}
void orc_set_backend(orc_ctx* c, void* m, void* s, void* r)
{
    if (m) c->match_fn = (match_lines_fn_t)m;
    if (s) c->score_fn = (score_matches_fn_t)s;
    if (r) c->rdd_fn = (rdd_fn_t)r;
}
void orc_set_match_source(orc_ctx* c, orc_match_source_fn fn) { c->match_source = fn; }
void orc_set_collinear_backend(orc_ctx* c, void* f) { c->collin_fn = f ? (collinear_fn_t)f : (collinear_fn_t)orc_collinear_f32; }

int orc_add_view(orc_ctx* c, uint32_t cam_id, int width, int height, const double* K, const double* R, const double* t,
                 float median_depth, const uint32_t* list, int n_list, const float* segs, int nseg)
{
    if (std::max(width, height) < 800) return -1;            // L3D_DEF_MIN_IMG_WIDTH line3D.cc:119
    if (c->views.count(cam_id)) return -2;                   // line3D.cc:130
    if (n_list == 0) return -3;                              // line3D.cc:154
    if (nseg == 0) return -4;
    View* v = new View(); v->id = cam_id; v->width = (unsigned)width; v->height = (unsigned)height;
    memcpy(v->K.m, K, 72); memcpy(v->R.m, R, 72); v->t = V(t[0], t[1], t[2]);
    v->initial_median_depth = (float)fmax(fabs((double)median_depth), L3D_EPS);
    v->lines.resize(nseg);
    for (int i = 0; i < nseg; ++i) { f4 l = {segs[4 * i], segs[4 * i + 1], segs[4 * i + 2], segs[4 * i + 3]}; v->lines[i] = l; }
    v->init();
    c->views[cam_id] = v; c->view_order.push_back(cam_id);
    c->matches[cam_id] = std::vector<std::list<orc_match_t> >(nseg);
    c->num_matches[cam_id] = 0; c->processed[cam_id] = false; c->visual_neighbors[cam_id] = std::set<uint32_t>();
    c->num_lines_total += nseg; c->views_avg_depths.push_back((float)fmax((double)median_depth, L3D_EPS));
    std::list<uint32_t> L(list, list + n_list);
    if (c->by_wps) { for (int i = 0; i < n_list; ++i) c->wps2views[list[i]].push_back(cam_id); c->num_wps[cam_id] = n_list; c->views2wps[cam_id] = L; }
    else c->fixed_neighbors[cam_id] = L;
    return 0;
}

int orc_match_images(orc_ctx* c, float sigma_position, float sigma_angle, uint32_t num_neighbors, float epipolar_overlap,
                     int kNN, float const_reg_depth)   // line3D.cc:375-497
{
    if (c->views.empty()) return -1;
    c->num_neighbors = (unsigned)std::max(int(num_neighbors), 2);
    c->sigma_p = sigma_position; c->sigma_a = fminf(fabsf(sigma_angle), 90.0f);
    c->two_sigA_sqr = 2.0f * c->sigma_a * c->sigma_a;
    c->epi = fminf(fabsf(epipolar_overlap), 0.99f); c->kNN = kNN; c->const_reg_depth = const_reg_depth;
    if (c->sigma_p < 0.0f) { c->fixed3Dreg = true; c->sigma_p = fabsf(c->sigma_p); }
    else { c->fixed3Dreg = false; c->sigma_p = fmaxf(0.1f, c->sigma_p); }
    c->matched.clear(); c->est.clear(); c->entry_map.clear(); c->pairs.clear(); c->pair_evals = 0; c->scored.clear();
    c->med_scene_depth = const_reg_depth;
    if (const_reg_depth < 0.0f && c->fixed3Dreg && !c->views_avg_depths.empty()) {
        std::sort(c->views_avg_depths.begin(), c->views_avg_depths.end());
        c->med_scene_depth = c->views_avg_depths[c->views_avg_depths.size() / 2];
    }
    translate(c);
    for (size_t i = 0; i < c->view_order.size(); ++i) {
        uint32_t cam = c->view_order[i]; View* v = c->views[cam];
        if (!c->fixed3Dreg) v->k = v->specificSpatialReg(c->sigma_p); else v->k = c->sigma_p / c->med_scene_depth;
        c->matches[cam] = std::vector<std::list<orc_match_t> >(v->lines.size());
        c->num_matches[cam] = 0; c->processed[cam] = false;
    }
    for (size_t i = 0; i < c->view_order.size(); ++i) {
        uint32_t cam = c->view_order[i];
        if (c->fixed_neighbors.count(cam)) {
            if (c->visual_neighbors[cam].empty())
                for (std::list<uint32_t>::const_iterator n = c->fixed_neighbors[cam].begin(); n != c->fixed_neighbors[cam].end(); ++n)
                    if (c->views.count(*n)) c->visual_neighbors[cam].insert(*n);
        } else find_visual_neighbors_from_wps(c, cam);
    }
    compute_matches(c);
    untranslate(c);
    return 0;
}

int orc_reconstruct_opt(orc_ctx* c, uint32_t visibility_t, int perform_diffusion, float collinearity_t, int use_ceres, uint32_t max_iter_ceres);
int orc_reconstruct(orc_ctx* c, uint32_t visibility_t, int perform_diffusion, float collinearity_t)
{ return orc_reconstruct_opt(c, visibility_t, perform_diffusion, collinearity_t, 0, 0); }

// Line3D::optimizeClusters (line3D.cc:2269-2275) -> LineOptimizer::optimize
static void optimize_clusters(orc_ctx* c, uint32_t max_iter)
{
    const int L = (int)c->clusters3D.size();
    if (L == 0) return;
    std::map<uint32_t, int> cam_local; std::vector<double> cams;
    for (std::map<uint32_t, View*>::const_iterator v = c->views.begin(); v != c->views.end(); ++v) {     // optimization.cc:106-142
        cam_local[v->first] = (int)cam_local.size();
        const View* w = v->second;
        for (int k = 0; k < 9; ++k) cams.push_back(w->R.m[k]);
        cams.push_back(w->C.x); cams.push_back(w->C.y); cams.push_back(w->C.z);
        cams.push_back(w->K(0, 0)); cams.push_back(w->K(1, 1)); cams.push_back(w->K(0, 2)); cams.push_back(w->K(1, 2));
    }
    std::vector<double> p((size_t)6 * L), xy; std::vector<long long> ptr((size_t)L + 1, 0); std::vector<int> rcam;
    for (int i = 0; i < L; ++i) {
        const Seg3D& s = c->clusters3D[i].cluster_seg;
        p[6 * i] = s.P1.x; p[6 * i + 1] = s.P1.y; p[6 * i + 2] = s.P1.z; p[6 * i + 3] = s.P2.x; p[6 * i + 4] = s.P2.y; p[6 * i + 5] = s.P2.z;
        for (std::list<Seg2D>::const_iterator it = c->clusters3D[i].residuals.begin(); it != c->clusters3D[i].residuals.end(); ++it) {
            const f4& ln = c->views[it->cam]->lines[it->seg];
            rcam.push_back(cam_local[it->cam]);
            xy.push_back(ln.x); xy.push_back(ln.y); xy.push_back(ln.z); xy.push_back(ln.w);
        }
        ptr[i + 1] = (long long)rcam.size();
    }
    std::vector<int> valid(L);
    orc_optimize_lines(L, p.data(), ptr.data(), rcam.data(), xy.data(), (int)cam_local.size(), cams.data(), (int)max_iter, p.data(), valid.data(), c->opt_summary);
    std::vector<FinalLine> kept;
    for (int i = 0; i < L; ++i) {
        if (!valid[i]) continue;
        c->clusters3D[i].cluster_seg = Seg3D(V(p[6 * i], p[6 * i + 1], p[6 * i + 2]), V(p[6 * i + 3], p[6 * i + 4], p[6 * i + 5]));
        kept.push_back(c->clusters3D[i]);
    }
    c->clusters3D = kept;
}

int orc_reconstruct_opt(orc_ctx* c, uint32_t visibility_t, int perform_diffusion, float collinearity_t, int use_ceres, uint32_t max_iter_ceres)   // line3D.cc:1702-1824
{
    if (c->est.empty()) return -1;
    c->visibility_t = (unsigned)std::max(int(visibility_t), 3);
    c->clusters3D.clear(); c->lines3D.clear();
    const float prev_collin_t = c->collin_t;
    c->collin_t = collinearity_t;
    c->perform_RDD = perform_diffusion && c->use_gpu;
    translate(c);
    if (c->collin_t > L3D_EPS && (prev_collin_t < L3D_EPS || std::fabs(prev_collin_t - c->collin_t) > L3D_EPS))   // line3D.cc:1751-1756, 1827-1849
        for (std::map<uint32_t, View*>::iterator v = c->views.begin(); v != c->views.end(); ++v) view_find_collinear(c, v->second, c->collin_t, c->use_gpu);
    std::vector<float> sd;
    for (std::map<uint32_t, View*>::const_iterator v = c->views.begin(); v != c->views.end(); ++v)
        if (v->second->median_depth > L3D_EPS) sd.push_back(v->second->median_depth);
    if (!sd.empty()) { std::sort(sd.begin(), sd.end()); c->med_scene_depth_lines = sd[sd.size() / 2]; } else c->med_scene_depth_lines = 0.0f;
    computing_affinity_matrix(c);
    c->A_raw = c->A;
    c->l2g_dump.clear();
    for (std::map<int, Seg2D>::const_iterator it = c->local2global.begin(); it != c->local2global.end(); ++it) c->l2g_dump.push_back(it->second);
    if (c->perform_RDD) perform_rdd(c);
    cluster_segments(c);
    c->global2local.clear(); c->local2global.clear();
    if (use_ceres) optimize_clusters(c, max_iter_ceres);        // line3D.cc:1800-1805
    for (size_t i = 0; i < c->clusters3D.size(); ++i) {   // computeFinal3Dsegments line3D.cc:2278-2299
        std::list<Seg3D> col = find_collinear_segments(c, c->clusters3D[i]);
        if (!col.empty()) { FinalLine f = c->clusters3D[i]; f.collinear = col; c->lines3D.push_back(f); }
    }
    c->clusters3D.clear();
    {   // filterTinySegments line3D.cc:2302-2339
        std::vector<FinalLine> kept;
        for (size_t i = 0; i < c->lines3D.size(); ++i) {
            View* v = c->views[c->lines3D[i].reference_view];
            std::list<Seg3D> f;
            for (std::list<Seg3D>::const_iterator it = c->lines3D[i].collinear.begin(); it != c->lines3D[i].collinear.end(); ++it)
                if (v->projectedLongEnough(*it)) f.push_back(*it);
            c->lines3D[i].collinear = f;
            if (!f.empty()) kept.push_back(c->lines3D[i]);
        }
        c->lines3D = kept;
    }
    untranslate(c);
    return 0;
}

int orc_get_opt_summary(orc_ctx* c, double* s8) { for (int k = 0; k < 8; ++k) s8[k] = c->opt_summary[k]; return 0; }
int orc_num_views(orc_ctx* c) { return (int)c->views.size(); }
long long orc_pair_evals(orc_ctx* c) { return c->pair_evals; }
int orc_get_pairs(orc_ctx* c, int* st, int cap)
{
    for (size_t i = 0; i < c->pairs.size() && (int)i < cap; ++i) { st[2 * i] = (int)c->pairs[i].first; st[2 * i + 1] = (int)c->pairs[i].second; }
    return (int)c->pairs.size();
}
long long orc_get_matches(orc_ctx* c, uint32_t cam, orc_match_t* out, long long cap)
{
    long long n = 0;
    if (!c->matches.count(cam)) return -1;
    const std::vector<std::list<orc_match_t> >& M = c->matches[cam];
    for (size_t i = 0; i < M.size(); ++i)
        for (std::list<orc_match_t>::const_iterator it = M[i].begin(); it != M[i].end(); ++it) { if (out && n < cap) out[n] = *it; ++n; }
    return n;
}
long long orc_get_scored(orc_ctx* c, uint32_t cam, orc_match_t* out, long long cap)
{
    if (!c->scored.count(cam)) return -1;
    const std::vector<orc_match_t>& d = c->scored[cam];
    for (size_t i = 0; i < d.size() && (long long)i < cap; ++i) if (out) out[i] = d[i];
    return (long long)d.size();
}
int orc_get_view_info(orc_ctx* c, uint32_t cam, float* k, float* md)
{
    if (!c->views.count(cam)) return -1;
    *k = c->views[cam]->k; *md = c->views[cam]->median_depth; return 0;
}
long long orc_get_estimates(orc_ctx* c, orc_match_t* best, double* p, long long cap)
{
    for (size_t i = 0; i < c->est.size() && (long long)i < cap; ++i) {
        if (best) best[i] = c->est[i].second;
        if (p) { const Seg3D& s = c->est[i].first; p[6 * i] = s.P1.x; p[6 * i + 1] = s.P1.y; p[6 * i + 2] = s.P1.z; p[6 * i + 3] = s.P2.x; p[6 * i + 4] = s.P2.y; p[6 * i + 5] = s.P2.z; }
    }
    return (long long)c->est.size();
}
static long long dump_edges(const std::list<CLEdge>& A, int* ei, int* ej, float* ew, long long cap)
{
    long long n = 0;
    for (std::list<CLEdge>::const_iterator it = A.begin(); it != A.end(); ++it, ++n) if (ei && n < cap) { ei[n] = it->i; ej[n] = it->j; ew[n] = it->w; }
    return n;
}
long long orc_get_affinity(orc_ctx* c, int* ei, int* ej, float* ew, long long cap) { return dump_edges(c->A_final, ei, ej, ew, cap); }
long long orc_get_affinity_raw(orc_ctx* c, int* ei, int* ej, float* ew, long long cap) { return dump_edges(c->A_raw, ei, ej, ew, cap); }
int orc_get_local2global(orc_ctx* c, uint32_t* cs, int cap)
{
    for (size_t i = 0; i < c->l2g_dump.size() && (int)i < cap; ++i) { cs[2 * i] = c->l2g_dump[i].cam; cs[2 * i + 1] = c->l2g_dump[i].seg; }
    return (int)c->l2g_dump.size();
}
// collinear lists of a view as CSR: row_ptr[nseg+1], idx[row_ptr[nseg]]; returns the number of entries (even if > cap)
long long orc_get_collinear(orc_ctx* c, uint32_t cam, long long* row_ptr, int* idx, long long cap)
{
    if (!c->views.count(cam)) return -1;
    View* v = c->views[cam];
    long long n = 0;
    for (size_t i = 0; i < v->lines.size(); ++i) {
        if (row_ptr) row_ptr[i] = n;
        if (i < v->collin.size())
            for (std::list<uint32_t>::const_iterator it = v->collin[i].begin(); it != v->collin[i].end(); ++it) { if (idx && n < cap) idx[n] = (int)*it; ++n; }
    }
    if (row_ptr) row_ptr[v->lines.size()] = n;
    return n;
}
// findCollinearSegments(cluster) (line3D.cc:2342-2452) on an explicit cluster: end points of the cluster line + (camID, segID)
// residuals of views added with orc_add_view.  Returns the number of 3D segments (out6: 6 doubles each).
int orc_collinear_from_cluster(orc_ctx* c, const double* p1p2, int nres, const uint32_t* cams, const uint32_t* segs, double* out6, int cap)
{
    FinalLine cl;
    cl.cluster_seg = Seg3D(V(p1p2[0], p1p2[1], p1p2[2]), V(p1p2[3], p1p2[4], p1p2[5]));
    for (int i = 0; i < nres; ++i) { Seg2D s = {cams[i], segs[i]}; cl.residuals.push_back(s); }
    cl.reference_view = nres ? cams[0] : 0;
    std::list<Seg3D> col = find_collinear_segments(c, cl);
    int n = 0;
    for (std::list<Seg3D>::const_iterator it = col.begin(); it != col.end(); ++it, ++n)
        if (n < cap) { double* o = out6 + 6 * n; o[0] = it->P1.x; o[1] = it->P1.y; o[2] = it->P1.z; o[3] = it->P2.x; o[4] = it->P2.y; o[5] = it->P2.z; }
    return n;
}
int orc_num_lines(orc_ctx* c) { return (int)c->lines3D.size(); }
long long orc_get_segments3d(orc_ctx* c, orc_seg3d_t* out, long long cap)
{
    long long n = 0;
    for (size_t i = 0; i < c->lines3D.size(); ++i)
        for (std::list<Seg3D>::const_iterator it = c->lines3D[i].collinear.begin(); it != c->lines3D[i].collinear.end(); ++it, ++n)
            if (out && n < cap) { out[n].line = (int)i; out[n].p1[0] = it->P1.x; out[n].p1[1] = it->P1.y; out[n].p1[2] = it->P1.z; out[n].p2[0] = it->P2.x; out[n].p2[1] = it->P2.y; out[n].p2[2] = it->P2.z; }
    return n;
}
long long orc_get_residuals(orc_ctx* c, orc_residual_t* out, long long cap)
{
    long long n = 0;
    for (size_t i = 0; i < c->lines3D.size(); ++i)
        for (std::list<Seg2D>::const_iterator it = c->lines3D[i].residuals.begin(); it != c->lines3D[i].residuals.end(); ++it, ++n)
            if (out && n < cap) { out[n].line = (int)i; out[n].cam = it->cam; out[n].seg = it->seg; }
    return n;
}
int orc_save_txt(orc_ctx* c, const char* path)   // line3D.cc:2650-2681
{
    std::ofstream f(path);
    if (!f) return -1;
    for (size_t i = 0; i < c->lines3D.size(); ++i) {
        const FinalLine& L = c->lines3D[i];
        if (L.collinear.empty()) continue;
        f << L.collinear.size() << " ";
        for (std::list<Seg3D>::const_iterator it = L.collinear.begin(); it != L.collinear.end(); ++it)
            f << it->P1.x << " " << it->P1.y << " " << it->P1.z << " " << it->P2.x << " " << it->P2.y << " " << it->P2.z << " ";
        f << L.residuals.size() << " ";
        for (std::list<Seg2D>::const_iterator it = L.residuals.begin(); it != L.residuals.end(); ++it) {
            f4 co = c->views[it->cam]->lines[it->seg];
            f << it->cam << " " << it->seg << " " << co.x << " " << co.y << " " << co.z << " " << co.w << " ";
        }
        f << std::endl;
    }
    return 0;
}

} // extern "C"
