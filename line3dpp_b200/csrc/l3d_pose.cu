// l3d_pose.cu — visual neighbours from camera poses alone (l3d_pose_neighbors, include/l3d_capi.h; DESIGN.md §6d).  Every view gets a
// grid of virtual world points: pixel samples back-projected to the view's median depth.  A point is observed by its own view and by
// every other view it projects into.  The neighbours are then what findVisualNeighborsFromWPs (line3D.cc:578-699) chooses for those
// points: the device computes the observations, the co-visibility counts and each view's ranked candidates; the host runs the
// selection of line3d_host.cc over the ranked candidates only.  Not part of the pipeline chain: no stage is touched.
#include "l3d_cub.cuh"
#include "l3d_pose_select.h"

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include <chrono>
#include <climits>
#include <cmath>
#include <string>
#include <unordered_map>

#define PS_THREADS 256
#define PO_THREADS 128
#define PO_TILE 64                     // views whose cameras a CTA of k_pose_observe stages in shared memory at once
#define PC_THREADS 512
#define PC_NOT_CANDIDATE 0xffffffffffffffffull   // rank key of a co-visible view with common <= 4: after every candidate

// one view as the kernels read it; all doubles, so that a tile is copied to shared memory as a flat array
struct PoseCam {
    double fx, fy, cx, cy, skew;
    double r[9], t[3];
    double w, h;                       // the image size (exact in double)
};
static_assert(sizeof(PoseCam) == 19 * sizeof(double), "PoseCam is staged as doubles");

// Step 2 of the definition (DESIGN.md §6d), in this order: u = ((c + 0.5) * width) / gx, v = ((r + 0.5) * height) / gy;
// yn = (v - cy) / fy, xn = ((u - cx) - skew * yn) / fx (K^-1 [u v 1] by back-substitution); q = (z * xn, z * yn, z) with
// z = median_depth; d = q - t; X_k = (R_0k d_0 + R_1k d_1) + R_2k d_2.  One thread per (view, sample); X in three planes.
__global__ void __launch_bounds__(PS_THREADS) k_pose_samples(long long P, int G, int gx, int gy, const PoseCam* __restrict__ cams,
                                                             const double* __restrict__ depth, double* __restrict__ X)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int i = (int)(p / G), s = (int)(p % G);
    const int r = s / gx, c = s % gx;
    const PoseCam& v = cams[i];
    const double u = ((double)c + 0.5) * v.w / (double)gx, vv = ((double)r + 0.5) * v.h / (double)gy;
    const double yn = (vv - v.cy) / v.fy;
    const double xn = ((u - v.cx) - v.skew * yn) / v.fx;
    const double z = depth[i];
    const double d0 = z * xn - v.t[0], d1 = z * yn - v.t[1], d2 = z - v.t[2];
    X[p] = (v.r[0] * d0 + v.r[3] * d1) + v.r[6] * d2;
    X[P + p] = (v.r[1] * d0 + v.r[4] * d1) + v.r[7] * d2;
    X[2 * P + p] = (v.r[2] * d0 + v.r[5] * d1) + v.r[8] * d2;
}

// Step 3: c = R X + t (each row ((R_k0 X + R_k1 Y) + R_k2 Z) + t_k), p = K c = ((fx c0 + skew c1) + cx c2, fy c1 + cy c2, c2); seen when
// c2 > 0, 0 <= p.x / c2 < width and 0 <= p.y / c2 < height.  No occlusion and no depth range.
__device__ __forceinline__ bool pose_sees(const PoseCam& v, double x, double y, double z)
{
    const double c2 = ((v.r[6] * x + v.r[7] * y) + v.r[8] * z) + v.t[2];
    if (!(c2 > 0.0)) return false;
    const double c0 = ((v.r[0] * x + v.r[1] * y) + v.r[2] * z) + v.t[0];
    const double c1 = ((v.r[3] * x + v.r[4] * y) + v.r[5] * z) + v.t[1];
    const double u = ((v.fx * c0 + v.skew * c1) + v.cx * c2) / c2;
    if (!(u >= 0.0 && u < v.w)) return false;
    const double vv = (v.fy * c1 + v.cy * c2) / c2;
    return vv >= 0.0 && vv < v.h;
}

// Every point against every view: one thread per point, the CTA walks the views in tiles of PO_TILE cameras staged in shared memory
// (every thread of a warp reads the same camera: a broadcast).  FILL = false: cnt[p] = the point's observers; FILL = true: its
// observers in ascending view order at obs[off[p]..], and p beside each of them in obs_pt.  A point's own view observes it.
template <bool FILL>
__global__ void __launch_bounds__(PO_THREADS) k_pose_observe(long long P, int n, int G, const PoseCam* __restrict__ cams, const double* __restrict__ X,
                                                             long long* __restrict__ cnt, const long long* __restrict__ off, int* __restrict__ obs,
                                                             int* __restrict__ obs_pt)
{
    __shared__ double s_cam[PO_TILE * 19];
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = p < P;
    const double x = live ? X[p] : 0.0, y = live ? X[P + p] : 0.0, z = live ? X[2 * P + p] : 0.0;
    const int own = live ? (int)(p / G) : -1;
    long long o = FILL && live ? off[p] : 0, k = 0;
    for (int v0 = 0; v0 < n; v0 += PO_TILE) {
        const int nv = min(PO_TILE, n - v0);
        __syncthreads();
        for (int e = threadIdx.x; e < nv * 19; e += blockDim.x) s_cam[e] = ((const double*)(cams + v0))[e];
        __syncthreads();
        if (!live) continue;
        const PoseCam* s = (const PoseCam*)s_cam;
        for (int j = 0; j < nv; ++j) {
            if (v0 + j == own || pose_sees(s[j], x, y, z)) {
                if (FILL) { obs[o + k] = v0 + j; obs_pt[o + k] = (int)p; }
                ++k;
            }
        }
    }
    if (!FILL && live) cnt[p] = k;
}

// per view: the first entry of its points in the view-sorted observation list (vkeys ascending); voff[n] = E
__global__ void k_pose_view_ranges(int n, long long E, const int* __restrict__ vkeys, long long* __restrict__ voff)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v > n) return;
    long long lo = 0, hi = E;
    while (lo < hi) {
        const long long mid = lo + (hi - lo) / 2;
        if (vkeys[mid] < v) lo = mid + 1; else hi = mid;
    }
    voff[v] = lo;
}

// per view i: a bound on its co-visible views, min(n - 1, sum over its points of (observers - 1)) (slots of k_pose_covis's output)
__global__ void __launch_bounds__(256) k_pose_bound(int n, const long long* __restrict__ voff, const int* __restrict__ vpts, const long long* __restrict__ off,
                                                    long long* __restrict__ bound)
{
    typedef cub::BlockReduce<long long, 256> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const int i = blockIdx.x;
    long long s = 0;
    for (long long e = voff[i] + threadIdx.x; e < voff[i + 1]; e += blockDim.x) {
        const int p = vpts[e];
        s += off[p + 1] - off[p] - 1;
    }
    s = Reduce(tmp).Sum(s);
    if (threadIdx.x == 0) bound[i] = min(s, (long long)(n - 1));
}

// Step 4 and the ranking: one CTA per view i, a shared histogram over all views.  A warp per point of i's list adds the point's
// observers (shared-memory atomics; exact integer counts, no global atomics); hist[i] is then n_i and hist[j] common(i, j).  The
// co-visible views j != i are written in ascending j at slots[i]..: j, common, and the rank key
// (~bits(score) << 32 | camID_j) for common > 4 (PC_NOT_CANDIDATE otherwise), score = 2.0f * float(common) / float(n_i + n_j) as
// find_visual_neighbors computes it.  Ascending keys: score descending, camID ascending.
__global__ void __launch_bounds__(PC_THREADS) k_pose_covis(int n, const long long* __restrict__ voff, const int* __restrict__ vpts,
                                                           const long long* __restrict__ off, const int* __restrict__ obs,
                                                           const uint32_t* __restrict__ cam_id, const long long* __restrict__ slots,
                                                           long long* __restrict__ seg_end, int* __restrict__ nz_j, int* __restrict__ nz_c,
                                                           unsigned long long* __restrict__ keys)
{
    extern __shared__ unsigned int hist[];
    typedef cub::BlockScan<int, PC_THREADS> Scan;
    __shared__ typename Scan::TempStorage scan_tmp;
    const int i = blockIdx.x;
    for (int j = threadIdx.x; j < n; j += blockDim.x) hist[j] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    for (long long e = voff[i] + warp; e < voff[i + 1]; e += warps) {
        const int p = vpts[e];
        for (long long q = off[p] + lane; q < off[p + 1]; q += 32) atomicAdd(&hist[obs[q]], 1u);
    }
    __syncthreads();
    const unsigned long long ni = hist[i];
    long long base = slots[i];
    for (int j0 = 0; j0 < n; j0 += blockDim.x) {
        const int j = j0 + threadIdx.x;
        const unsigned int c = (j < n && j != i) ? hist[j] : 0u;
        int pos, total;
        Scan(scan_tmp).ExclusiveSum(c > 0 ? 1 : 0, pos, total);
        if (c > 0) {
            const long long slot = base + pos;
            nz_j[slot] = j;
            nz_c[slot] = (int)c;
            unsigned long long key = PC_NOT_CANDIDATE;
            if (c > 4) {
                const unsigned long long nj = (unsigned long long)(voff[j + 1] - voff[j]);
                const float score = 2.0f * __uint2float_rn(c) / __ull2float_rn(ni + nj);
                key = ((unsigned long long)(0xffffffffu - __float_as_uint(score)) << 32) | cam_id[j];
            }
            keys[slot] = key;
        }
        base += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) seg_end[i] = base;
}

// ------------------------------------------------------------------------------------------------ host side
namespace {

std::string view_name(const l3d_pose_view& v, int i) { return "view " + std::to_string(i) + " (camID " + std::to_string(v.cam_id) + ")"; }

// the checks of l3d_pose_neighbors: "" or the reason
std::string check_pose_views(int n, const l3d_pose_view* views, int gx, int gy)
{
    if (n < 0) return "n < 0";
    if (n > 0 && !views) return "no view array";
    if (gx < 1 || gy < 1) return "gx and gy must be at least 1 (gx = " + std::to_string(gx) + ", gy = " + std::to_string(gy) + ")";
    std::unordered_map<uint32_t, int> seen;
    for (int i = 0; i < n; ++i) {
        const l3d_pose_view& v = views[i];
        if (!(v.median_depth > 0.0) || !std::isfinite(v.median_depth)) return view_name(v, i) + ": median_depth must be finite and > 0";
        if (v.width < 1 || v.height < 1) return view_name(v, i) + ": width and height must be at least 1";
        if (!(v.fx != 0.0) || !std::isfinite(v.fx) || !(v.fy != 0.0) || !std::isfinite(v.fy)) return view_name(v, i) + ": fx or fy is zero or not finite";
        if (!std::isfinite(v.cx) || !std::isfinite(v.cy) || !std::isfinite(v.skew)) return view_name(v, i) + ": cx, cy or skew is not finite";
        bool finite = true;
        for (int k = 0; k < 9; ++k) finite = finite && std::isfinite(v.R[k]);
        if (!finite) return view_name(v, i) + ": R is not finite";
        for (int k = 0; k < 3; ++k) finite = finite && std::isfinite(v.t[k]);
        if (!finite) return view_name(v, i) + ": t is not finite";
        const auto ins = seen.emplace(v.cam_id, i);
        if (!ins.second) return view_name(v, i) + ": duplicate camID, already view " + std::to_string(ins.first->second);
    }
    if (n > L3D_POSE_MAX_VIEWS) return "more than L3D_POSE_MAX_VIEWS (" + std::to_string(L3D_POSE_MAX_VIEWS) + ") views";
    if ((long long)n * gx * gy > L3D_POSE_MAX_POINTS || (long long)gx * gy > L3D_POSE_MAX_POINTS)
        return "n * gx * gy above L3D_POSE_MAX_POINTS (" + std::to_string(L3D_POSE_MAX_POINTS) + ")";
    return "";
}

// What both entry points compute on the device and download: per view n_obs (n_i) and its co-visible views (slot range [slots[i],
// slots[i] + nz[i]) of nz_j / nz_c), the rank keys sorted within each view (keys), and the device time of the phases.
struct PoseResult {
    std::vector<long long> voff, slots, seg_end;
    std::vector<int> nz_j, nz_c;
    std::vector<unsigned long long> keys;
    float device_ms = 0.f;
};

int pose_device(l3d_ctx* c, const char* what, int n, const l3d_pose_view* views, int gx, int gy, bool want_pairs, PoseResult& res)
{
    const int G = gx * gy;
    const long long P = (long long)n * G;
    std::vector<PoseCam> hc((size_t)n);
    std::vector<double> hd((size_t)n);
    std::vector<uint32_t> hid((size_t)n);
    for (int i = 0; i < n; ++i) {
        const l3d_pose_view& v = views[i];
        PoseCam& q = hc[i];
        q.fx = v.fx; q.fy = v.fy; q.cx = v.cx; q.cy = v.cy; q.skew = v.skew;
        for (int k = 0; k < 9; ++k) q.r[k] = v.R[k];
        for (int k = 0; k < 3; ++k) q.t[k] = v.t[k];
        q.w = (double)v.width; q.h = (double)v.height;
        hd[i] = v.median_depth; hid[i] = v.cam_id;
    }
    cudaSetDevice(c->device);
    int rc;
    DevBuf d_cams, d_depth, d_id, d_X, d_cnt, d_off, d_obs, d_obspt, d_vkeys, d_vpts, d_voff, d_bound, d_slots, d_end, d_nzj, d_nzc, d_keys, d_keys2;
    L3D_RESERVE(d_cams, sizeof(PoseCam) * (size_t)n, "pose cameras");
    L3D_RESERVE(d_depth, sizeof(double) * (size_t)n, "pose depths");
    L3D_RESERVE(d_id, sizeof(uint32_t) * (size_t)n, "pose camIDs");
    L3D_RESERVE(d_X, 3 * sizeof(double) * (size_t)P, "virtual points");
    L3D_RESERVE(d_cnt, sizeof(long long) * (size_t)(P + 1), "observer counts");
    L3D_RESERVE(d_off, sizeof(long long) * (size_t)(P + 1), "observer offsets");
    L3D_CUDA(c, cudaMemcpyAsync(d_cams.p, hc.data(), sizeof(PoseCam) * (size_t)n, cudaMemcpyHostToDevice, c->stream), "pose upload");
    L3D_CUDA(c, cudaMemcpyAsync(d_depth.p, hd.data(), sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, c->stream), "pose upload");
    L3D_CUDA(c, cudaMemcpyAsync(d_id.p, hid.data(), sizeof(uint32_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream), "pose upload");
    L3D_CUDA(c, cudaMemsetAsync((long long*)d_cnt.p + P, 0, sizeof(long long), c->stream), "observer counts");
    ScopedEvent e0, e1;
    if ((rc = e0.create(c)) || (rc = e1.create(c))) return rc;
    L3D_CUDA(c, cudaEventRecord(e0.e, c->stream), "event");

    const PoseCam* cams = (const PoseCam*)d_cams.p;
    double* X = (double*)d_X.p;
    long long* cnt = (long long*)d_cnt.p;
    long long* off = (long long*)d_off.p;
    k_pose_samples<<<(unsigned)((P + PS_THREADS - 1) / PS_THREADS), PS_THREADS, 0, c->stream>>>(P, G, gx, gy, cams, (const double*)d_depth.p, X);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_pose_samples");
    const unsigned po_blocks = (unsigned)((P + PO_THREADS - 1) / PO_THREADS);
    k_pose_observe<false><<<po_blocks, PO_THREADS, 0, c->stream>>>(P, n, G, cams, X, cnt, nullptr, nullptr, nullptr);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_pose_observe (count)");
    if ((rc = l3d_cub(c, "observer offsets", [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, cnt, off, P + 1, c->stream); })))
        return rc;
    long long E = 0;
    L3D_CUDA(c, cudaMemcpyAsync(&E, off + P, sizeof(long long), cudaMemcpyDeviceToHost, c->stream), "observation count");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "observation count");
    if (E > INT_MAX) return l3d_fail(c, L3D_ERR_UNSUPPORTED, (std::string(what) + ": more than 2^31 - 1 observations of virtual points").c_str());
    L3D_RESERVE(d_obs, sizeof(int) * (size_t)E, "observers");
    L3D_RESERVE(d_obspt, sizeof(int) * (size_t)E, "observed points");
    L3D_RESERVE(d_vkeys, sizeof(int) * (size_t)E, "observers by view");
    L3D_RESERVE(d_vpts, sizeof(int) * (size_t)E, "points by view");
    L3D_RESERVE(d_voff, sizeof(long long) * ((size_t)n + 1), "view offsets");
    k_pose_observe<true><<<po_blocks, PO_THREADS, 0, c->stream>>>(P, n, G, cams, X, nullptr, off, (int*)d_obs.p, (int*)d_obspt.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_pose_observe (fill)");
    // the transposed list: every view's observed points, ascending (a stable sort of the point-ordered list by view)
    int bits = 1;
    while ((1ll << bits) < n) ++bits;
    if ((rc = l3d_cub(c, "points by view", [&](void* tmp, size_t& bytes) {
             return cub::DeviceRadixSort::SortPairs(tmp, bytes, (const int*)d_obs.p, (int*)d_vkeys.p, (const int*)d_obspt.p, (int*)d_vpts.p, (int)E, 0, bits,
                                                    c->stream);
         })))
        return rc;
    long long* voff = (long long*)d_voff.p;
    k_pose_view_ranges<<<(unsigned)((n + 1 + 127) / 128), 128, 0, c->stream>>>(n, E, (const int*)d_vkeys.p, voff);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_pose_view_ranges");
    L3D_RESERVE(d_bound, sizeof(long long) * ((size_t)n + 1), "co-visibility bounds");
    L3D_RESERVE(d_slots, sizeof(long long) * ((size_t)n + 1), "co-visibility slots");
    L3D_RESERVE(d_end, sizeof(long long) * (size_t)n, "co-visibility ends");
    long long* bound = (long long*)d_bound.p;
    L3D_CUDA(c, cudaMemsetAsync(bound + n, 0, sizeof(long long), c->stream), "co-visibility bounds");
    k_pose_bound<<<(unsigned)n, 256, 0, c->stream>>>(n, voff, (const int*)d_vpts.p, off, bound);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_pose_bound");
    long long* slots = (long long*)d_slots.p;
    if ((rc = l3d_cub(c, "co-visibility slots", [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, bound, slots, n + 1, c->stream); })))
        return rc;
    long long S = 0;
    L3D_CUDA(c, cudaMemcpyAsync(&S, slots + n, sizeof(long long), cudaMemcpyDeviceToHost, c->stream), "co-visibility slots");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "co-visibility slots");
    if (S > INT_MAX) return l3d_fail(c, L3D_ERR_UNSUPPORTED, (std::string(what) + ": more than 2^31 - 1 co-visibility slots").c_str());
    L3D_RESERVE(d_nzj, sizeof(int) * (size_t)S, "co-visible views");
    L3D_RESERVE(d_nzc, sizeof(int) * (size_t)S, "co-visibility counts");
    L3D_RESERVE(d_keys, sizeof(unsigned long long) * (size_t)S, "rank keys");
    L3D_RESERVE(d_keys2, sizeof(unsigned long long) * (size_t)S, "sorted rank keys");
    const size_t smem = sizeof(unsigned int) * (size_t)n;
    L3D_CUDA(c, cudaFuncSetAttribute(k_pose_covis, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1)), "k_pose_covis smem");
    k_pose_covis<<<(unsigned)n, PC_THREADS, smem, c->stream>>>(n, voff, (const int*)d_vpts.p, off, (const int*)d_obs.p, (const uint32_t*)d_id.p, slots,
                                                               (long long*)d_end.p, (int*)d_nzj.p, (int*)d_nzc.p, (unsigned long long*)d_keys.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_pose_covis");
    if (S > 0 &&
        (rc = l3d_cub(c, "rank sort", [&](void* tmp, size_t& bytes) {
             return cub::DeviceSegmentedSort::SortKeys(tmp, bytes, (const unsigned long long*)d_keys.p, (unsigned long long*)d_keys2.p, (int)S, n, slots,
                                                       (const long long*)d_end.p, c->stream);
         })))
        return rc;
    L3D_CUDA(c, cudaEventRecord(e1.e, c->stream), "event");
    res.voff.resize((size_t)n + 1); res.slots.resize((size_t)n + 1); res.seg_end.resize((size_t)n); res.keys.resize((size_t)S);
    L3D_CUDA(c, cudaMemcpyAsync(res.voff.data(), voff, sizeof(long long) * ((size_t)n + 1), cudaMemcpyDeviceToHost, c->stream), "pose download");
    L3D_CUDA(c, cudaMemcpyAsync(res.slots.data(), slots, sizeof(long long) * ((size_t)n + 1), cudaMemcpyDeviceToHost, c->stream), "pose download");
    L3D_CUDA(c, cudaMemcpyAsync(res.seg_end.data(), d_end.p, sizeof(long long) * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "pose download");
    if (S > 0) L3D_CUDA(c, cudaMemcpyAsync(res.keys.data(), d_keys2.p, sizeof(unsigned long long) * (size_t)S, cudaMemcpyDeviceToHost, c->stream), "pose download");
    if (want_pairs && S > 0) {
        res.nz_j.resize((size_t)S); res.nz_c.resize((size_t)S);
        L3D_CUDA(c, cudaMemcpyAsync(res.nz_j.data(), d_nzj.p, sizeof(int) * (size_t)S, cudaMemcpyDeviceToHost, c->stream), "pose download");
        L3D_CUDA(c, cudaMemcpyAsync(res.nz_c.data(), d_nzc.p, sizeof(int) * (size_t)S, cudaMemcpyDeviceToHost, c->stream), "pose download");
    }
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "pose download");
    L3D_CUDA(c, cudaEventElapsedTime(&res.device_ms, e0.e, e1.e), "event");
    return L3D_OK;
}

int pose_prologue(l3d_ctx* c, const char* what, int n, const l3d_pose_view* views, int gx, int gy)
{
    const std::string why = check_pose_views(n, views, gx, gy);
    if (why.empty()) return L3D_OK;
    const bool big = why.find("L3D_POSE_MAX") != std::string::npos;
    return l3d_fail(c, big ? L3D_ERR_UNSUPPORTED : L3D_ERR_INVALID, (std::string(what) + ": " + why).c_str());
}

}  // namespace

extern "C" {

long long l3d_pose_neighbors(l3d_ctx* c, int n, const l3d_pose_view* views, int gx, int gy, unsigned int num_neighbors, int64_t* nb_ptr, uint32_t* nb_cam,
                             long long cap, int32_t* n_obs_out, double* timing_out)
{
    if (!c) return L3D_ERR_INVALID;
    int rc;
    if ((rc = pose_prologue(c, "l3d_pose_neighbors", n, views, gx, gy))) return rc;
    if (!nb_ptr) return l3d_fail(c, L3D_ERR_INVALID, "l3d_pose_neighbors: no nb_ptr array");
    nb_ptr[0] = 0;
    if (n == 0) return 0;
    PoseResult r;
    if ((rc = pose_device(c, "l3d_pose_neighbors", n, views, gx, gy, false, r))) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    // each view's candidates, ranked: the keys up to the first PC_NOT_CANDIDATE of its sorted segment
    std::vector<long long> cand_off((size_t)n + 1, 0);
    std::vector<L3DPP::PoseCandidate> cand;
    for (int i = 0; i < n; ++i) {
        for (long long s = r.slots[i]; s < r.seg_end[i] && r.keys[s] != PC_NOT_CANDIDATE; ++s) {
            const unsigned long long k = r.keys[s];
            L3DPP::PoseCandidate pc;
            pc.cam = (unsigned int)(k & 0xffffffffu);
            const unsigned int bits = 0xffffffffu - (unsigned int)(k >> 32);
            memcpy(&pc.score, &bits, sizeof(float));
            cand.push_back(pc);
        }
        cand_off[i + 1] = (long long)cand.size();
    }
    std::vector<std::vector<unsigned int> > nb;
    L3DPP::pose_select_neighbors(n, views, cand_off.data(), cand.data(), num_neighbors, nb);
    long long total = 0;
    for (int i = 0; i < n; ++i) { total += (long long)nb[i].size(); nb_ptr[i + 1] = total; }
    if (nb_cam && total <= cap)
        for (int i = 0; i < n; ++i) std::copy(nb[i].begin(), nb[i].end(), nb_cam + nb_ptr[i]);
    if (n_obs_out)
        for (int i = 0; i < n; ++i) n_obs_out[i] = (int32_t)(r.voff[i + 1] - r.voff[i]);
    if (timing_out) {
        timing_out[0] = r.device_ms;
        timing_out[1] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    return total;
}

long long l3d_pose_covisibility(l3d_ctx* c, int n, const l3d_pose_view* views, int gx, int gy, int32_t* n_obs_out, int32_t* ijc_out, long long cap)
{
    if (!c) return L3D_ERR_INVALID;
    int rc;
    if ((rc = pose_prologue(c, "l3d_pose_covisibility", n, views, gx, gy))) return rc;
    if (n == 0) return 0;
    PoseResult r;
    if ((rc = pose_device(c, "l3d_pose_covisibility", n, views, gx, gy, true, r))) return rc;
    long long total = 0;
    for (int i = 0; i < n; ++i) total += r.seg_end[i] - r.slots[i];
    if (n_obs_out)
        for (int i = 0; i < n; ++i) n_obs_out[i] = (int32_t)(r.voff[i + 1] - r.voff[i]);
    if (ijc_out && total <= cap) {
        long long t = 0;
        for (int i = 0; i < n; ++i)
            for (long long s = r.slots[i]; s < r.seg_end[i]; ++s, ++t) {
                ijc_out[3 * t] = i; ijc_out[3 * t + 1] = r.nz_j[s]; ijc_out[3 * t + 2] = r.nz_c[s];
            }
    }
    return total;
}

}  // extern "C"
