// l3d_triangulate.cu — linear triangulation of tie points and per-camera median depths: the host loops of the reference's Pix4D
// frontend (main_pix4d.cpp:34-70 linearHomTriangulation, 354-372 the loop over every point, 386-418 the median depth of every
// camera) as the two C-ABI entries l3d_triangulate_points / l3d_median_depths of include/l3d_capi.h.  The arithmetic contract is
// DESIGN.md §6b.  Like the undistortion calls, neither entry belongs to the pipeline: they never drop a stage and touch only the
// buffers of TriangulateState and, in host mode, the context's staging pair.
#include "l3d_cub.cuh"

#include <cub/device/device_segmented_sort.cuh>

#include <climits>
#include <cmath>
#include <cstring>

#define TR_THREADS 128
#define TR_SMEM_MAX (96 * 1024)         // camera matrices are staged in shared memory up to this size (1024 cameras)
#define TR_EPS 2.220446049250313e-16    // DBL_EPSILON: a Jacobi rotation is skipped when |a_pq| <= TR_EPS * sqrt(|a_pp|) * sqrt(|a_qq|)
#define TR_MAX_SWEEPS 32
#define TR_L3D_EPS 1e-12                // L3D_EPS (commons.h:95): the reference's validity threshold on |X|
#define MD_THREADS 256
#define MD_INVALID 0xffffffffu          // sort key of a list entry whose point is not valid: above the bits of every depth

// One cyclic-Jacobi rotation of the symmetric 4x4 matrix a that zeroes a[p][q]; V accumulates the rotations (its columns become
// the eigenvectors).  The rotation of Numerical Recipes §11.1 (t = the smaller root, tau = s / (1 + c)).  Returns whether it
// rotated.  A NaN element is never rotated on, so a non-finite matrix ends the sweeps instead of looping.
template <int p, int q>
__host__ __device__ __forceinline__ bool tr_rotate(double (&a)[4][4], double (&V)[4][4])
{
    const double apq = a[p][q];
    if (!(fabs(apq) > TR_EPS * (sqrt(fabs(a[p][p])) * sqrt(fabs(a[q][q]))))) return false;
    const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
    double t = fabs(theta) > 1e150 ? 0.5 / fabs(theta) : 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
    if (theta < 0.0) t = -t;
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c), h = t * apq;
    a[p][p] = a[p][p] - h;
    a[q][q] = a[q][q] + h;
    a[p][q] = a[q][p] = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        if (r == p || r == q) continue;
        const double g = a[r][p], k = a[r][q];
        a[r][p] = a[p][r] = g - s * (k + g * tau);
        a[r][q] = a[q][r] = k + s * (g - k * tau);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const double g = V[r][p], k = V[r][q];
        V[r][p] = g - s * (k + g * tau);
        V[r][q] = k + s * (g - k * tau);
    }
    return true;
}

// the unit eigenvector of the smallest eigenvalue of the symmetric 4x4 matrix a (a is overwritten): cyclic Jacobi in the fixed
// order (0,1) (0,2) (0,3) (1,2) (1,3) (2,3) until a sweep rotates nothing (at most TR_MAX_SWEEPS sweeps); ties of the diagonal
// pick the lower index
__host__ __device__ __forceinline__ void tr_smallest_eigvec(double (&a)[4][4], double v[4])
{
    double V[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) V[r][c] = r == c ? 1.0 : 0.0;
    for (int sweep = 0; sweep < TR_MAX_SWEEPS; ++sweep) {
        bool rot = tr_rotate<0, 1>(a, V);
        rot = tr_rotate<0, 2>(a, V) || rot;
        rot = tr_rotate<0, 3>(a, V) || rot;
        rot = tr_rotate<1, 2>(a, V) || rot;
        rot = tr_rotate<1, 3>(a, V) || rot;
        rot = tr_rotate<2, 3>(a, V) || rot;
        if (!rot) break;
    }
    double best = a[0][0];              // compile-time indices only, so that a and V stay in registers
#pragma unroll
    for (int r = 0; r < 4; ++r) v[r] = V[r][0];
#pragma unroll
    for (int i = 1; i < 4; ++i)
        if (a[i][i] < best) {
            best = a[i][i];
#pragma unroll
            for (int r = 0; r < 4; ++r) v[r] = V[r][i];
        }
}

// A^T A of linearHomTriangulation: per observation the rows Sx * P[cam] (main_pix4d.cpp:45-51), Sx = [[0,-1,y],[1,0,-x]], added in
// observation order.  Returns false when an observation names a camera outside [0, n_cams).
__host__ __device__ __forceinline__ bool tr_normal_matrix(long long b, long long e, const int32_t* cam, const double* xy, int n_cams, const double* P,
                                                          double (&a)[4][4])
{
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) a[r][c] = 0.0;
    for (long long o = b; o < e; ++o) {
        const int ci = cam[o];
        if ((unsigned)ci >= (unsigned)n_cams) return false;
        const double x = xy[2 * o], y = xy[2 * o + 1];
        const double* M = P + 12 * (long long)ci;
        double r1[4], r2[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            r1[j] = -M[4 + j] + y * M[8 + j];
            r2[j] = M[j] - x * M[8 + j];
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = r; c < 4; ++c) a[r][c] = a[r][c] + (r1[r] * r1[c] + r2[r] * r2[c]);
    }
#pragma unroll
    for (int r = 1; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < r; ++c) a[r][c] = a[c][r];
    return true;
}

// one point: fewer than three observations (main_pix4d.cpp:363) or an unknown camera -> invalid with X = 0 (the reference leaves
// feat_pos3D at 0); otherwise X = v.xyz / v.w and valid = |X| > L3D_EPS as the reference compares it (NaN invalid, +-Inf valid)
__host__ __device__ __forceinline__ int tr_point(long long b, long long e, const int32_t* cam, const double* xy, int n_cams, const double* P, double X[3])
{
    X[0] = X[1] = X[2] = 0.0;
    if (e - b < 3) return 0;
    double a[4][4], v[4];
    if (!tr_normal_matrix(b, e, cam, xy, n_cams, P, a)) return 0;
    tr_smallest_eigvec(a, v);
    X[0] = v[0] / v[3]; X[1] = v[1] / v[3]; X[2] = v[2] / v[3];
    return sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]) > TR_L3D_EPS ? 1 : 0;
}

// One thread per point, grid-stride.  staged != 0: the camera matrices are copied to shared memory once per CTA (the grid is then
// one resident wave) and gathered from there; otherwise they are read from global memory.  Consecutive threads take consecutive
// CSR rows, so a warp's observation reads fall in one contiguous stretch of the arrays.
__global__ void __launch_bounds__(TR_THREADS) k_triangulate(long long n, const long long* __restrict__ ptr, const int32_t* __restrict__ cam,
                                                            const double* __restrict__ xy, int n_cams, const double* __restrict__ P, int staged,
                                                            double* __restrict__ X, int32_t* __restrict__ valid)
{
    extern __shared__ double s_P[];
    const double* M = P;
    if (staged) {
        for (int i = threadIdx.x; i < 12 * n_cams; i += blockDim.x) s_P[i] = P[i];
        __syncthreads();
        M = s_P;
    }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        double x[3];
        valid[i] = tr_point(ptr[i], ptr[i + 1], cam, xy, n_cams, M, x);
        X[3 * i] = x[0]; X[3 * i + 1] = x[1]; X[3 * i + 2] = x[2];
    }
}

// sort keys of the median pass: one CTA per camera; the bits of the float depth |X - C| (main_pix4d.cpp:397-402, a double norm stored
// as float) of every valid point of the camera's list, MD_INVALID for the others (and for ids outside [0, n_points)).  A depth is +0,
// positive or +inf, never NaN (a valid X has a finite or infinite norm), and the bits of such floats sort as unsigned integers in the
// order of their values, so the sort compares no floats.
__global__ void __launch_bounds__(MD_THREADS) k_depth_keys(const long long* __restrict__ lptr, const int32_t* __restrict__ lpts, long long n_points,
                                                           const double* __restrict__ X, const int32_t* __restrict__ valid, const double* __restrict__ C,
                                                           unsigned int* __restrict__ keys)
{
    const int cam = blockIdx.x;
    const double cx = C[3 * cam], cy = C[3 * cam + 1], cz = C[3 * cam + 2];
    for (long long e = lptr[cam] + threadIdx.x; e < lptr[cam + 1]; e += blockDim.x) {
        const int p = lpts[e];
        unsigned int k = MD_INVALID;
        if (p >= 0 && p < n_points && valid[p]) {
            const double dx = X[3 * p] - cx, dy = X[3 * p + 1] - cy, dz = X[3 * p + 2] - cz;
            k = __float_as_uint((float)sqrt(dx * dx + dy * dy + dz * dz));
        }
        keys[e] = k;
    }
}

// per camera: the number of valid entries (they sort before every MD_INVALID key) and the element at count/2 of their sorted depths
__global__ void k_pick_median(int n_cams, const long long* __restrict__ lptr, const unsigned int* __restrict__ sorted, int32_t* __restrict__ count,
                              float* __restrict__ median)
{
    const int cam = blockIdx.x * blockDim.x + threadIdx.x;
    if (cam >= n_cams) return;
    const long long b = lptr[cam];
    long long lo = b, hi = lptr[cam + 1];          // first MD_INVALID key in [lo, hi)
    while (lo < hi) {
        const long long mid = lo + (hi - lo) / 2;
        if (sorted[mid] == MD_INVALID) hi = mid; else lo = mid + 1;
    }
    const long long n = lo - b;
    count[cam] = (int32_t)n;
    median[cam] = n ? __uint_as_float(sorted[b + n / 2]) : 0.0f;
}

// ------------------------------------------------------------------------------------------------ host side
extern "C" {

int l3d_triangulate_points(l3d_ctx* c, long long n_points, const int64_t* obs_ptr, const int32_t* obs_cam, const double* obs_xy, int n_cams,
                           const double* P, double* X_out, int32_t* valid_out, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (n_points < 0 || n_cams < 0 || !obs_ptr || !X_out || !valid_out || (n_cams && !P))
        return l3d_fail(c, L3D_ERR_INVALID, "l3d_triangulate_points: bad arguments");
    if (n_points == 0) return L3D_OK;
    cudaSetDevice(c->device);
    int rc;
    const long long* ptr = (const long long*)obs_ptr;
    const int32_t* cam = obs_cam;
    const double* xy = obs_xy;
    const double* Pd = P;
    double* X = X_out;
    int32_t* valid = valid_out;
    HostBlock out[2] = {host_array(X_out, 3 * sizeof(double) * (size_t)n_points), host_array(valid_out, sizeof(int32_t) * (size_t)n_points)};
    if (!on_device) {       // host arrays are checked here; on the device an unknown camera makes its point invalid
        if (obs_ptr[0] != 0) return l3d_fail(c, L3D_ERR_INVALID, "l3d_triangulate_points: obs_ptr[0] must be 0");
        for (long long i = 0; i < n_points; ++i)
            if (obs_ptr[i + 1] < obs_ptr[i]) return l3d_fail(c, L3D_ERR_INVALID, "l3d_triangulate_points: obs_ptr must not decrease");
        const long long n_obs = obs_ptr[n_points];
        if (n_obs && (!obs_cam || !obs_xy)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_triangulate_points: null observation arrays");
        for (long long o = 0; o < n_obs; ++o)
            if (obs_cam[o] < 0 || obs_cam[o] >= n_cams) return l3d_fail(c, L3D_ERR_INVALID, "l3d_triangulate_points: observation of an unknown camera");
        HostBlock in[4] = {host_array(obs_ptr, sizeof(long long) * ((size_t)n_points + 1)), host_array(obs_cam, sizeof(int32_t) * (size_t)n_obs),
                           host_array(obs_xy, 2 * sizeof(double) * (size_t)n_obs), host_array(P, 12 * sizeof(double) * (size_t)n_cams)};
        if ((rc = l3d_stage_host(c, in, 4, out, 2))) return rc;
        ptr = (const long long*)in[0].dev; cam = (const int32_t*)in[1].dev; xy = (const double*)in[2].dev; Pd = (const double*)in[3].dev;
        X = (double*)out[0].dev; valid = (int32_t*)out[1].dev;
    }
    const size_t smem = 12 * sizeof(double) * (size_t)n_cams;
    const int staged = n_cams > 0 && smem <= TR_SMEM_MAX;
    long long blocks = (n_points + TR_THREADS - 1) / TR_THREADS;
    if (staged) {
        L3D_CUDA(c, cudaFuncSetAttribute(k_triangulate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "k_triangulate smem");
        int per_sm = 0;
        L3D_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_triangulate, TR_THREADS, smem), "k_triangulate occupancy");
        blocks = std::min<long long>(blocks, (long long)c->num_sms * std::max(per_sm, 1));
    }
    blocks = std::min<long long>(blocks, INT_MAX);
    k_triangulate<<<(unsigned)blocks, TR_THREADS, staged ? smem : 0, c->stream>>>(n_points, ptr, cam, xy, n_cams, Pd, staged, X, valid);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_triangulate");
    if (!on_device && (rc = l3d_unstage_host(c, out, 2, "l3d_triangulate_points"))) return rc;
    return L3D_OK;
}

int l3d_median_depths(l3d_ctx* c, int n_cams, const int64_t* list_ptr, const int32_t* list_pts, long long n_points, const double* X, const int32_t* valid,
                      const double* C, int32_t* count_out, float* median_out, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (n_cams < 0 || n_points < 0 || !list_ptr || !count_out || !median_out || (n_cams && !C) || (n_points && (!X || !valid)))
        return l3d_fail(c, L3D_ERR_INVALID, "l3d_median_depths: bad arguments");
    if (n_cams == 0) return L3D_OK;
    cudaSetDevice(c->device);
    TriangulateState& s = c->tri;
    int rc;
    long long total = 0;
    const long long* lptr = (const long long*)list_ptr;
    const int32_t* lpts = list_pts;
    const double *Xd = X, *Cd = C;
    const int32_t* vd = valid;
    int32_t* cnt = count_out;
    float* med = median_out;
    HostBlock out[2] = {host_array(count_out, sizeof(int32_t) * (size_t)n_cams), host_array(median_out, sizeof(float) * (size_t)n_cams)};
    if (!on_device) {
        if (list_ptr[0] != 0) return l3d_fail(c, L3D_ERR_INVALID, "l3d_median_depths: list_ptr[0] must be 0");
        for (int i = 0; i < n_cams; ++i)
            if (list_ptr[i + 1] < list_ptr[i]) return l3d_fail(c, L3D_ERR_INVALID, "l3d_median_depths: list_ptr must not decrease");
        total = list_ptr[n_cams];
        if (total && !list_pts) return l3d_fail(c, L3D_ERR_INVALID, "l3d_median_depths: null point list");
        for (long long e = 0; e < total; ++e)
            if (list_pts[e] < 0 || list_pts[e] >= n_points) return l3d_fail(c, L3D_ERR_INVALID, "l3d_median_depths: point id out of range");
        HostBlock in[5] = {host_array(list_ptr, sizeof(long long) * ((size_t)n_cams + 1)), host_array(list_pts, sizeof(int32_t) * (size_t)total),
                           host_array(X, 3 * sizeof(double) * (size_t)n_points), host_array(valid, sizeof(int32_t) * (size_t)n_points),
                           host_array(C, 3 * sizeof(double) * (size_t)n_cams)};
        if ((rc = l3d_stage_host(c, in, 5, out, 2))) return rc;
        lptr = (const long long*)in[0].dev; lpts = (const int32_t*)in[1].dev; Xd = (const double*)in[2].dev; vd = (const int32_t*)in[3].dev;
        Cd = (const double*)in[4].dev;
        cnt = (int32_t*)out[0].dev; med = (float*)out[1].dev;
    } else {
        L3D_CUDA(c, cudaMemcpyAsync(&total, list_ptr + n_cams, sizeof(long long), cudaMemcpyDeviceToHost, c->stream), "list length");
        L3D_CUDA(c, cudaStreamSynchronize(c->stream), "list length");
    }
    if (total < 0 || total > INT_MAX) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_median_depths: more than 2^31 - 1 list entries in one call");
    if (n_cams > INT_MAX / 2) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_median_depths: too many cameras");
    L3D_RESERVE(s.d_keys, sizeof(unsigned int) * (size_t)total, "depth keys");
    L3D_RESERVE(s.d_keys2, sizeof(unsigned int) * (size_t)total, "sorted depth keys");
    k_depth_keys<<<(unsigned)n_cams, MD_THREADS, 0, c->stream>>>(lptr, lpts, n_points, Xd, vd, Cd, (unsigned int*)s.d_keys.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_depth_keys");
    if (total > 0) {
        if ((rc = l3d_cub(c, "median depth sort", [&](void* tmp, size_t& bytes) {
                 return cub::DeviceSegmentedSort::SortKeys(tmp, bytes, (const unsigned int*)s.d_keys.p, (unsigned int*)s.d_keys2.p, (int)total, n_cams, lptr, lptr + 1,
                                                           c->stream);
             })))
            return rc;
    }
    k_pick_median<<<(unsigned)((n_cams + 127) / 128), 128, 0, c->stream>>>(n_cams, lptr, (const unsigned int*)s.d_keys2.p, cnt, med);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_pick_median");
    if (!on_device && (rc = l3d_unstage_host(c, out, 2, "l3d_median_depths"))) return rc;
    return L3D_OK;
}

} // extern "C"
