// l3d_cub.cuh — cub calls on the context's stream and scratch buffer
#pragma once
#include "l3d_ctx.cuh"

#include <cub/device/device_scan.cuh>

// A two-phase cub call f(tmp, bytes): the size query with tmp == nullptr, then the call on c->cub_tmp.
template <class F> int l3d_cub(l3d_ctx* c, const char* what, F&& f)
{
    size_t bytes = 0;
    L3D_CUDA(c, f(nullptr, bytes), what);
    int rc;
    if ((rc = c->cub_tmp.reserve(c, bytes, what))) return rc;
    L3D_CUDA(c, f(c->cub_tmp.p, bytes), what);
    return L3D_OK;
}

// The total of an exclusive scan `out` over n items is out[n-1] plus the last item, which is computed from src[n-1].
// l3d_read_total queues the downloads of both; they are valid once the caller has synchronised the stream.
struct ScanTotal { long long last_out = 0; int last_src = 0; };
inline int l3d_read_total(l3d_ctx* c, const long long* out, const int* src, long long n, ScanTotal& t, const char* what)
{
    L3D_CUDA(c, cudaMemcpyAsync(&t.last_out, out + n - 1, sizeof(long long), cudaMemcpyDeviceToHost, c->stream), what);
    L3D_CUDA(c, cudaMemcpyAsync(&t.last_src, src + n - 1, sizeof(int), cudaMemcpyDeviceToHost, c->stream), what);
    return L3D_OK;
}

// exclusive sum of `n` items of `in` into `out`, then l3d_read_total
template <class In, class N>
int l3d_scan_total(l3d_ctx* c, In in, long long* out, N n, const int* src, ScanTotal& t, const char* what)
{
    int rc;
    if ((rc = l3d_cub(c, what, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, n, c->stream); }))) return rc;
    return l3d_read_total(c, out, src, (long long)n, t, what);
}
