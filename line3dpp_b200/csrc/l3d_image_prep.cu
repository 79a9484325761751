// l3d_image_prep.cu — the image the reference's detectLineSegments hands to LSD (line3D.cc:249-289): cvtColor(CV_RGB2GRAY) for
// 3-channel input, then cv::resize(gray, out, Size(), s, s) with INTER_LINEAR when max_img_width asks for it, fused into one kernel
// over a batch of images; and the two C-ABI entry points declared in include/l3d_capi.h.  The arithmetic contract is DESIGN.md §4b;
// tests/image_prep_model.py restates it.
//
// None of these calls belongs to the pipeline: they never drop a stage and touch only the buffers of ImagePrepState and, in host
// mode, the context's staging pair.
#include "l3d_ctx.cuh"
#include "../../include/line3d_io.h"   // preparedImageSize: the one rounding of the prepared size (csrc/line3d_bin.cc)

#include <cstring>

#define PR_TW 128       // destination columns per tile of k_prepare_gray_u8 (one per thread)
#define PR_TH 8         // destination rows per tile

#define L3D_PREP_COPY 0     // no resize: grey conversion (or a copy) only
#define L3D_PREP_LINEAR 1   // INTER_LINEAR downscale
#define L3D_PREP_AREA2 2    // source step exactly 2: OpenCV's fast INTER_AREA 2x2 mean

#define PR_COEF 2048        // INTER_RESIZE_COEF_SCALE

// RGB2Gray<uchar> of one source pixel: channel 0 is R, 15-bit fixed point, rounded
template <int C>
__device__ __forceinline__ int pr_gray(const unsigned char* __restrict__ p)
{
    if (C == 1) return __ldg(p);
    return ((int)__ldg(p) * 9798 + (int)__ldg(p + 1) * 19235 + (int)__ldg(p + 2) * 3735 + (1 << 14)) >> 15;
}

// OpenCV's interpolation taps of destination index d when downscaling (resize.cpp, the xofs / ialpha and yofs / ibeta tables):
// f = (float)((d + 0.5) * scale - 0.5) in double, first tap cvFloor(f), weights saturate_cast<short>((1 - frac) * 2048) and
// saturate_cast<short>(frac * 2048) in float
__device__ __forceinline__ void pr_taps(int d, double scale, int& i, int& w0, int& w1)
{
    float f = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
    i = (int)floorf(f);
    f = __fsub_rn(f, (float)i);
    w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), (float)PR_COEF));
    w1 = __float2int_rn(__fmul_rn(f, (float)PR_COEF));
}

// one destination pixel (column j, row i); x0 / x1 / a0 / a1: the column's source byte offsets and weights (linear), x0: the block's
// first byte (area), x0: the pixel's byte (copy)
template <int C, int MODE>
__device__ __forceinline__ unsigned char pr_pixel(const L3DPrepImage& d, int j, int i, long long x0, long long x1, int a0, int a1)
{
    const unsigned char* __restrict__ src = d.src;
    if (MODE == L3D_PREP_COPY) return (unsigned char)pr_gray<C>(src + (long long)i * d.src_pitch + x0);
    if (MODE == L3D_PREP_LINEAR) {
        // vertical taps: both rows clamped into the image, the weights kept (resizeGeneric_Invoker's clip)
        int sy, b0, b1;
        pr_taps(i, d.scale, sy, b0, b1);
        const unsigned char* p0 = src + (long long)max(0, min(sy, d.height - 1)) * d.src_pitch;
        const unsigned char* p1 = src + (long long)max(0, min(sy + 1, d.height - 1)) * d.src_pitch;
        const int S0 = pr_gray<C>(p0 + x0) * a0 + pr_gray<C>(p0 + x1) * a1;
        const int S1 = pr_gray<C>(p1 + x0) * a0 + pr_gray<C>(p1 + x1) * a1;
        // VResizeLinearVec_32s8u: v_mul_hi of (S >> 4) with the weights, saturating add, rounding shift by 2, pack to 8 bits
        const int v = (((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16);
        return (unsigned char)min(255, (v + 2) >> 2);
    }
    const int sx = 2 * j, sy = 2 * i;
    const unsigned char* p = src + (long long)sy * d.src_pitch + x0;
    if (sx + 2 <= d.width && sy + 2 <= d.height)
        return (unsigned char)((pr_gray<C>(p) + pr_gray<C>(p + C) + pr_gray<C>(p + d.src_pitch) + pr_gray<C>(p + d.src_pitch + C) + 2) >> 2);
    // resizeAreaFast_'s border: the mean of the block's pixels inside the image, (float)sum / count, cvRound
    int sum = 0, count = 0;
    for (int dy = 0; dy < 2 && sy + dy < d.height; ++dy)
        for (int dx = 0; dx < 2 && sx + dx < d.width; ++dx) { sum += pr_gray<C>(p + (long long)dy * d.src_pitch + dx * C); ++count; }
    return (unsigned char)min(255, max(0, __float2int_rn(__fdiv_rn((float)sum, (float)count))));
}

// one destination column j, rows [i0, i0 + rows): every row's value first, then the stores, so that the rows' loads overlap
template <int C, int MODE>
__device__ __forceinline__ void pr_column(const L3DPrepImage& d, int j, int i0, int rows)
{
    long long x0 = (long long)j * C, x1 = x0;
    int a0 = PR_COEF, a1 = 0;
    if (MODE == L3D_PREP_LINEAR) {
        // horizontal taps; a column whose second tap leaves the image takes its first (clamped) at full weight
        int sx;
        pr_taps(j, d.scale, sx, a0, a1);
        if (sx + 1 >= d.width) { sx = min(sx, d.width - 1); a0 = PR_COEF; a1 = 0; }
        x0 = (long long)sx * C; x1 = (long long)min(sx + 1, d.width - 1) * C;
    } else if (MODE == L3D_PREP_AREA2) {
        x0 = 2ll * j * C;
    }
    unsigned char v[PR_TH];
#pragma unroll
    for (int r = 0; r < PR_TH; ++r)
        if (r < rows) v[r] = pr_pixel<C, MODE>(d, j, i0 + r, x0, x1, a0, a1);
    unsigned char* out = d.dst + (long long)i0 * d.dst_pitch + j;
#pragma unroll
    for (int r = 0; r < PR_TH; ++r)
        if (r < rows) out[(long long)r * d.dst_pitch] = v[r];
}

// The fused path over a batch.  One CTA = PR_TW columns x PR_TH rows of one prepared image; the tiles of all images form one grid
// (image found by binary search over tile0), whatever their sizes, channel counts and modes.
__global__ void __launch_bounds__(PR_TW) k_prepare_gray_u8(const L3DPrepImage* __restrict__ imgs, int n)
{
    const L3DPrepImage d = imgs[last_le(n, (long long)blockIdx.x, [&](int i) { return imgs[i].tile0; })];
    const long long t = (long long)blockIdx.x - d.tile0;
    const int i0 = (int)(t / d.tiles_x) * PR_TH, j = (int)(t % d.tiles_x) * PR_TW + threadIdx.x;
    if (j >= d.out_w) return;
    const int rows = min(PR_TH, d.out_h - i0);
    const int key = d.mode * 4 + d.channels;
    switch (key) {
    case L3D_PREP_COPY * 4 + 1:   pr_column<1, L3D_PREP_COPY>(d, j, i0, rows); break;
    case L3D_PREP_COPY * 4 + 3:   pr_column<3, L3D_PREP_COPY>(d, j, i0, rows); break;
    case L3D_PREP_LINEAR * 4 + 1: pr_column<1, L3D_PREP_LINEAR>(d, j, i0, rows); break;
    case L3D_PREP_LINEAR * 4 + 3: pr_column<3, L3D_PREP_LINEAR>(d, j, i0, rows); break;
    case L3D_PREP_AREA2 * 4 + 1:  pr_column<1, L3D_PREP_AREA2>(d, j, i0, rows); break;
    default:                      pr_column<3, L3D_PREP_AREA2>(d, j, i0, rows); break;
    }
}

// ------------------------------------------------------------------------------------------------ host side
static int pr_check(l3d_ctx* c, const l3d_image_prep_desc& u)
{
    char buf[200];
    auto bad = [&](const char* why) { snprintf(buf, sizeof(buf), "l3d_prepare_gray_u8: %s", why); return l3d_fail(c, L3D_ERR_INVALID, buf); };
    if (u.width < 1 || u.width > 32767 || u.height < 1 || u.height > 32767) return bad("width and height must lie in [1, 32767]");
    if (u.channels != 1 && u.channels != 3) return bad("channels must be 1 or 3");
    int ow, oh;
    L3DPP::preparedImageSize(u.width, u.height, u.max_img_width, ow, oh);
    if (u.out_width != ow || u.out_height != oh) {
        snprintf(buf, sizeof(buf), "l3d_prepare_gray_u8: out size %dx%d, but l3d_image_prep_size gives %dx%d", u.out_width, u.out_height, ow, oh);
        return l3d_fail(c, L3D_ERR_INVALID, buf);
    }
    if (u.src_pitch < (long long)u.width * u.channels || u.dst_pitch < u.out_width) return bad("row pitch below the row's bytes");
    if (!u.src || !u.dst) return bad("null image pointer");
    if ((const void*)u.src == (const void*)u.dst) return bad("src == dst (no in-place preparation)");
    return L3D_OK;
}

// kernel parameters of one image (its size already checked)
static L3DPrepImage pr_image(const l3d_image_prep_desc& u, const unsigned char* src, long long src_pitch, unsigned char* dst, long long dst_pitch)
{
    L3DPrepImage d;
    memset(&d, 0, sizeof(d));
    d.src = src; d.dst = dst; d.src_pitch = src_pitch; d.dst_pitch = dst_pitch;
    d.width = u.width; d.height = u.height; d.channels = u.channels;
    float s = 1.0f;
    const bool resized = L3DPP::preparedImageSize(u.width, u.height, u.max_img_width, d.out_w, d.out_h, &s);
    // cv::resize's scale_x = 1. / inv_scale_x with inv_scale_x = (double)s; a step of exactly 2 switches INTER_LINEAR to INTER_AREA
    d.scale = resized ? 1.0 / (double)s : 1.0;
    d.mode = !resized ? L3D_PREP_COPY : (d.scale == 2.0 ? L3D_PREP_AREA2 : L3D_PREP_LINEAR);
    d.tiles_x = (d.out_w + PR_TW - 1) / PR_TW;
    return d;
}

extern "C" {

int l3d_image_prep_size(int width, int height, int max_img_width, int32_t* out_width, int32_t* out_height)
{
    if (!out_width || !out_height || width < 1 || width > 32767 || height < 1 || height > 32767) return L3D_ERR_INVALID;
    int ow, oh;
    const bool resized = L3DPP::preparedImageSize(width, height, max_img_width, ow, oh);
    *out_width = ow; *out_height = oh;
    return resized ? 1 : 0;
}

int l3d_prepare_gray_u8(l3d_ctx* c, int n, const l3d_image_prep_desc* descs, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (n < 0 || (n && !descs)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_prepare_gray_u8: bad arguments");
    for (int i = 0; i < n; ++i) {
        int rc = pr_check(c, descs[i]);
        if (rc) return rc;
    }
    if (n == 0) return L3D_OK;
    cudaSetDevice(c->device);
    ImagePrepState& s = c->prep;
    int rc;
    std::vector<HostBlock> in, out;         // host mode: every source and output
    if (!on_device) {
        for (int i = 0; i < n; ++i) {
            const l3d_image_prep_desc& u = descs[i];
            in.push_back({u.src, (size_t)u.src_pitch, (size_t)u.width * u.channels, (size_t)u.height});
            out.push_back({u.dst, (size_t)u.dst_pitch, (size_t)u.out_width, (size_t)u.out_height});
        }
        if ((rc = l3d_stage_host(c, in.data(), n, out.data(), n))) return rc;
    }
    s.h_imgs.resize(n);
    long long tiles = 0;
    for (int i = 0; i < n; ++i) {
        const l3d_image_prep_desc& u = descs[i];
        if (on_device) s.h_imgs[i] = pr_image(u, u.src, u.src_pitch, u.dst, u.dst_pitch);
        else s.h_imgs[i] = pr_image(u, (const unsigned char*)in[i].dev, (long long)in[i].row_bytes, (unsigned char*)out[i].dev, (long long)out[i].row_bytes);
        s.h_imgs[i].tile0 = tiles;
        tiles += (long long)s.h_imgs[i].tiles_x * ((u.out_height + PR_TH - 1) / PR_TH);
    }
    if (tiles >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_prepare_gray_u8: more than 2^31 tiles in one call");
    L3D_RESERVE(s.d_imgs, sizeof(L3DPrepImage) * (size_t)n, "image preparation descriptors");
    // pageable host memory: the copy is staged before the call returns, so h_imgs may be rewritten by the next call right away
    L3D_CUDA(c, cudaMemcpyAsync(s.d_imgs.p, s.h_imgs.data(), sizeof(L3DPrepImage) * n, cudaMemcpyHostToDevice, c->stream), "upload descriptors");
    k_prepare_gray_u8<<<(unsigned int)tiles, PR_TW, 0, c->stream>>>((const L3DPrepImage*)s.d_imgs.p, n);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_prepare_gray_u8");
    if (!on_device && (rc = l3d_unstage_host(c, out.data(), n, "l3d_prepare_gray_u8"))) return rc;
    return L3D_OK;
}

} // extern "C"
