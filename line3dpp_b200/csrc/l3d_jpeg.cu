// l3d_jpeg.cu — imread(path, IMREAD_GRAYSCALE) of a batch of JPEG files on the GPU, and its C-ABI entry point l3d_decode_jpeg_gray_u8
// (include/l3d_capi.h).  The host parses the markers (line3d_jpeg.cc); two kernels do the rest, each one launch for the whole batch:
//   k_jpeg_entropy  one thread per entropy-coded segment (a restart interval, or the whole scan): Huffman decoding of Y's scan, with
//                   un-stuffing, the DC predictors and their resets; Y's quantised coefficients go to a device buffer, chroma blocks
//                   of an interleaved scan are decoded and dropped.  Latency-bound per thread: the parallelism is the batch's segments.
//   k_jpeg_idct     one thread per 8x8 block that holds image pixels: dequantisation and the accurate integer IDCT as OpenCV's
//                   libjpeg-turbo computes it on x86 (its SIMD jsimd_idct_islow: 16-bit lanes, saturating packs), each pixel stored
//                   once at its place after the EXIF orientation.
// The arithmetic contract is DESIGN.md §4c; tests/jpeg_model.py restates it.  Not a pipeline stage: only JpegState's buffers and, in host
// mode, the context's staging pair change.
#include "l3d_ctx.cuh"
#include "l3d_exif.h"
#include "l3d_jpeg.h"

#include <climits>
#include <cstdio>
#include <cstring>

#define JP_IDCT_THREADS 128

__device__ const unsigned char c_jp_zigzag[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                                                  6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                                                  38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// status of an image after k_jpeg_entropy (JpegState::h_status)
#define JP_OK 0
#define JP_BAD_CODE 1       // no Huffman code matches the next 16 bits
#define JP_BAD_AC 2         // a run of AC coefficients passes index 63
#define JP_SHORT 3          // a segment needs more bits than it has

// ------------------------------------------------------------------------------------------------ entropy decoding
// MSB-first bit reader over one segment.  The host cut the data at its markers, so inside [p, end) a 0xFF is a stuffed data byte:
// the 0x00 after it (and any fill bytes between) are skipped.  Past the end it reads zero bytes and counts them in `pad`.
struct JpBits {
    const unsigned char* p;
    const unsigned char* end;
    unsigned long long buf;
    int n, pad;

    __device__ __forceinline__ void fill()
    {
        while (n <= 56) {
            unsigned int b = 0;
            if (p < end) {
                b = __ldg(p++);
                if (b == 0xFF) {
                    while (__ldg(p) == 0xFF) ++p;
                    ++p;
                }
            } else {
                pad += 8;
            }
            buf |= (unsigned long long)b << (56 - n);
            n += 8;
        }
    }
    __device__ __forceinline__ unsigned int peek(int k) const { return (unsigned int)(buf >> (64 - k)); }   // 1 <= k <= 32
    __device__ __forceinline__ void skip(int k) { buf <<= k; n -= k; }
};

// the next symbol of table t, -1 if no code matches; needs 16 bits in the reader
__device__ __forceinline__ int jp_symbol(JpBits& b, const L3DJpegTable* __restrict__ t)
{
    const unsigned int look = __ldg(&t->look[b.peek(9)]);
    if (look) { b.skip(look >> 8); return look & 255; }
    for (int l = 10; l <= 16; ++l) {
        const int code = (int)b.peek(l);
        if (code <= __ldg(&t->maxcode[l])) { b.skip(l); return __ldg(&t->vals[code + __ldg(&t->valoff[l])]); }
    }
    return -1;
}

// s value bits as a signed coefficient (HUFF_EXTEND); s = 0 is 0
__device__ __forceinline__ int jp_value(JpBits& b, int s)
{
    if (s == 0) return 0;
    const int v = (int)b.peek(s);
    b.skip(s);
    return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v;
}

// One thread per segment.  per_warp threads of each 32-thread CTA work (1..32): few segments are spread one per warp, so that no
// two long streams share a warp's issue slots; many are packed.
__global__ void __launch_bounds__(32) k_jpeg_entropy(const L3DJpegSeg* __restrict__ segs, int nseg, int per_warp, const L3DJpegImage* __restrict__ imgs,
                                                     const L3DJpegTable* __restrict__ tabs, const unsigned char* __restrict__ bytes,
                                                     short* __restrict__ coefs, int* __restrict__ status)
{
    if ((int)threadIdx.x >= per_warp) return;
    const int s = blockIdx.x * per_warp + threadIdx.x;
    if (s >= nseg) return;
    const L3DJpegSeg sg = segs[s];
    const L3DJpegImage* im = imgs + sg.image;
    const int ns = im->ns, yk = im->y_in_scan, mx = im->mcus_x, ybh = im->bh[yk], ybv = im->bv[yk], ybx = im->yblocks_x;
    const long long coef0 = im->coef0;
    const L3DJpegTable* tb = tabs + 8ll * sg.image;
    JpBits b;
    b.p = bytes + sg.first; b.end = bytes + sg.end; b.buf = 0; b.n = 0; b.pad = 0;
    int pred0 = 0, pred1 = 0, pred2 = 0, pred3 = 0;     // the DC predictors of the scan's components (named: no local-memory array)
    int err = JP_OK;
    for (int m = sg.mcu0; m < sg.mcu1 && err == JP_OK; ++m) {
        const int my = m / mx, mxx = m - my * mx;
        for (int k = 0; k < ns && err == JP_OK; ++k) {
            const int nb = im->bh[k] * im->bv[k];
            const L3DJpegTable* dct = tb + 2 * k;
            for (int i = 0; i < nb && err == JP_OK; ++i) {
                short* blk = nullptr;
                if (k == yk) {
                    const long long by = (long long)my * ybv + i / ybh, bx = (long long)mxx * ybh + i % ybh;
                    blk = coefs + (coef0 + by * ybx + bx) * 64;
                    int4* b4 = (int4*)blk;
#pragma unroll
                    for (int z = 0; z < 8; ++z) b4[z] = make_int4(0, 0, 0, 0);
                }
                if (b.n < 32) b.fill();
                const int sdc = jp_symbol(b, dct);
                if (sdc < 0) { err = JP_BAD_CODE; break; }
                const int dcv = jp_value(b, sdc);
                const int pred = (k == 0 ? pred0 : k == 1 ? pred1 : k == 2 ? pred2 : pred3) + dcv;
                if (k == 0) pred0 = pred; else if (k == 1) pred1 = pred; else if (k == 2) pred2 = pred; else pred3 = pred;
                if (blk) blk[0] = (short)pred;        // JCOEF: the predictor is an int, the stored coefficient its low 16 bits
                for (int z = 1; z < 64;) {
                    if (b.n < 32) b.fill();
                    const int rs = jp_symbol(b, dct + 1);
                    if (rs < 0) { err = JP_BAD_CODE; break; }
                    const int r = rs >> 4, sz = rs & 15;
                    if (sz) {
                        z += r;
                        if (z > 63) { err = JP_BAD_AC; break; }
                        const int v = jp_value(b, sz);
                        if (blk) blk[c_jp_zigzag[z]] = (short)v;
                        ++z;
                    } else if (r == 15) {
                        z += 16;
                    } else {
                        break;
                    }
                }
            }
        }
    }
    if (err == JP_OK && b.n < b.pad) err = JP_SHORT;     // some of the zero bits read past the end were used
    if (err != JP_OK) atomicMax(status + sg.image, err);
}

// ------------------------------------------------------------------------------------------------ IDCT
#define JP_CONST_BITS 13
#define JP_PASS1_BITS 2

__device__ __forceinline__ int jp_i16(int x) { return (int)(short)x; }
__device__ __forceinline__ int jp_sat16(int x) { return max(-32768, min(32767, x)); }

// one pass of jpeg_idct_islow in the SIMD code's form (pmaddwd pairs, 16-bit sums where it adds words): in[0..7] are 16-bit values,
// out[0..7] = the eight results descaled by `shift` and saturated to 16 bits.  Every 32-bit sum stays below 2^31.
__device__ __forceinline__ void jp_idct_1d(const int* in, int* out, int shift)
{
    const int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137, F1961 = 16069,
              F2053 = 16819, F2562 = 20995, F3072 = 25172;
    const int tmp2 = in[2] * F0541 + in[6] * (F0541 - F1847);
    const int tmp3 = in[2] * (F0541 + F0765) + in[6] * F0541;
    const int tmp0 = jp_i16(in[0] + in[4]) * (1 << JP_CONST_BITS);
    const int tmp1 = jp_i16(in[0] - in[4]) * (1 << JP_CONST_BITS);
    const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    const int z3 = jp_i16(in[7] + in[3]), z4 = jp_i16(in[5] + in[1]);
    const int Z3 = z3 * (F1175 - F1961) + z4 * F1175;
    const int Z4 = z3 * F1175 + z4 * (F1175 - F0390);
    const int T0 = in[7] * (F0298 - F0899) + in[1] * -F0899 + Z3;
    const int T3 = in[7] * -F0899 + in[1] * (F1501 - F0899) + Z4;
    const int T1 = in[5] * (F2053 - F2562) + in[3] * -F2562 + Z4;
    const int T2 = in[5] * -F2562 + in[3] * (F3072 - F2562) + Z3;
    const int round = 1 << (shift - 1);
    out[0] = jp_sat16((t10 + T3 + round) >> shift);
    out[7] = jp_sat16((t10 - T3 + round) >> shift);
    out[1] = jp_sat16((t11 + T2 + round) >> shift);
    out[6] = jp_sat16((t11 - T2 + round) >> shift);
    out[2] = jp_sat16((t12 + T1 + round) >> shift);
    out[5] = jp_sat16((t12 - T1 + round) >> shift);
    out[3] = jp_sat16((t13 + T0 + round) >> shift);
    out[4] = jp_sat16((t13 - T0 + round) >> shift);
}

// One thread per 8x8 block with image pixels; the blocks of all images form one grid (image found by binary search over tile0).
__global__ void __launch_bounds__(JP_IDCT_THREADS) k_jpeg_idct(const L3DJpegImage* __restrict__ imgs, int n, long long total,
                                                              const short* __restrict__ coefs)
{
    const long long t = (long long)blockIdx.x * JP_IDCT_THREADS + threadIdx.x;
    if (t >= total) return;
    const L3DJpegImage* im = imgs + last_le(n, t, [&](int i) { return imgs[i].tile0; });
    const long long local = t - im->tile0;
    const int by = (int)(local / im->blocks_x), bx = (int)(local % im->blocks_x);
    const int4* src = (const int4*)(coefs + (im->coef0 + (long long)by * im->yblocks_x + bx) * 64);
    const uint4* q4 = (const uint4*)im->q;
    int c[64];
    bool dc_only = true;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int4 v = __ldg(src + r);
        const uint4 qq = __ldg(q4 + r);
        const int w[4] = {v.x, v.y, v.z, v.w};
        const unsigned int qw[4] = {qq.x, qq.y, qq.z, qq.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // pmullw: the low 16 bits of coefficient * table entry
            c[8 * r + 2 * k] = jp_i16((int)(short)(w[k] & 0xFFFF) * (int)(qw[k] & 0xFFFF));
            c[8 * r + 2 * k + 1] = jp_i16((int)(short)((unsigned int)w[k] >> 16) * (int)(qw[k] >> 16));
        }
        if (r > 0) dc_only = dc_only && (v.x | v.y | v.z | v.w) == 0;
    }
    // pass 1 over columns into ws (row-major); the whole block takes the DC-only shortcut (a 16-bit shift) when rows 1..7 are zero
    int ws[64];
#pragma unroll
    for (int col = 0; col < 8; ++col) {
        int in[8], out[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) in[r] = c[8 * r + col];
        jp_idct_1d(in, out, JP_CONST_BITS - JP_PASS1_BITS);
#pragma unroll
        for (int r = 0; r < 8; ++r) ws[8 * r + col] = dc_only ? jp_i16(c[col] * (1 << JP_PASS1_BITS)) : out[r];
    }
    // pass 2 over rows, then packsswb's saturation and the +128 centring; every pixel inside the image goes to its oriented place
    const int y0 = by * 8, x0 = bx * 8;
    const int ryy = im->ryy, ryx = im->ryx, ry0 = im->ry0, rxy = im->rxy, rxx = im->rxx, rx0 = im->rx0;
    unsigned char* dst = im->dst;
    const long long pitch = im->dst_pitch;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        int out[8];
        jp_idct_1d(ws + 8 * r, out, JP_CONST_BITS + JP_PASS1_BITS + 3);
        const int y = y0 + r;
        if (y >= im->height) break;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int x = x0 + k;
            if (x < im->width)
                dst[(long long)(ryy * y + ryx * x + ry0) * pitch + (rxy * y + rxx * x + rx0)] = (unsigned char)(max(-128, min(127, out[k])) + 128);
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
static void jp_table(const L3DJpegHuffSpec& s, L3DJpegTable& t)
{
    memset(&t, 0, sizeof(t));
    memcpy(t.vals, s.vals, sizeof(t.vals));
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        t.valoff[l] = k - code;
        for (int i = 0; i < s.bits[l - 1]; ++i, ++code, ++k)
            if (l <= 9)
                for (int e = code << (9 - l); e < (code + 1) << (9 - l); ++e) t.look[e] = (unsigned short)(l << 8 | s.vals[k]);
        t.maxcode[l] = s.bits[l - 1] ? code - 1 : -1;
        code <<= 1;
    }
    t.maxcode[17] = 0x7FFFFFFF;
}

// the orientation as an affine map of (y, x) in a width x height frame (OpenCV's ExifTransform)
static void jp_orientation(L3DJpegImage& d, int o)
{
    int a[6];
    l3d_orientation_map(o, d.width, d.height, a);
    d.ryy = a[0]; d.ryx = a[1]; d.ry0 = a[2]; d.rxy = a[3]; d.rxx = a[4]; d.rx0 = a[5];
}

extern "C" int l3d_decode_jpeg_gray_u8(l3d_ctx* c, int n, const l3d_jpeg_desc* descs, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (n < 0 || (n && !descs)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_decode_jpeg_gray_u8: bad arguments");
    // every descriptor is checked (and every file parsed) before anything is launched
    std::vector<L3DJpegHeader> hdr(n);
    char buf[512];
    for (int i = 0; i < n; ++i) {
        const l3d_jpeg_desc& u = descs[i];
        std::string err;
        if (!u.data || u.size <= 0) err = "no file data";
        else if (!l3d_jpeg_parse(u.data, u.size, hdr[i], err)) {}
        else if (!u.dst) err = "null dst";
        else if (u.out_width != hdr[i].out_width || u.out_height != hdr[i].out_height) {
            snprintf(buf, sizeof(buf), "out size %dx%d, but l3d_jpeg_info gives %dx%d", u.out_width, u.out_height, hdr[i].out_width, hdr[i].out_height);
            err = buf;
        } else if (u.dst_pitch < u.out_width) err = "dst pitch below out_width";
        if (!err.empty()) {
            snprintf(buf, sizeof(buf), "l3d_decode_jpeg_gray_u8: image %d: %s", i, err.c_str());
            return l3d_fail(c, L3D_ERR_INVALID, buf);
        }
    }
    if (n == 0) return L3D_OK;
    cudaSetDevice(c->device);
    JpegState& s = c->jpeg;
    int rc;
    // sizes: Y's scan bytes, Y's coded blocks, the blocks with pixels, segments
    size_t bytes = 0;
    long long coef_blocks = 0, tiles = 0;
    size_t nseg = 0;
    for (int i = 0; i < n; ++i) {
        const L3DJpegHeader& h = hdr[i];
        bytes += (size_t)(h.segs.back().second - h.segs.front().first);
        coef_blocks += (long long)h.yblocks_x * h.yblocks_y;
        tiles += (long long)((h.width + 7) / 8) * ((h.height + 7) / 8);
        nseg += h.segs.size();
    }
    if (nseg > (size_t)INT_MAX || (tiles + JP_IDCT_THREADS - 1) / JP_IDCT_THREADS >= (1ll << 31))
        return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_decode_jpeg_gray_u8: too many segments or blocks in one call");
    L3D_RESERVE(s.d_bytes, bytes, "JPEG data staging");
    L3D_RESERVE(s.d_coefs, (size_t)coef_blocks * 128, "JPEG coefficients");
    L3D_RESERVE(s.d_status, sizeof(int) * (size_t)n, "JPEG status");
    std::vector<HostBlock> out;             // host mode: every output
    if (!on_device) {
        for (int i = 0; i < n; ++i) out.push_back({descs[i].dst, (size_t)descs[i].dst_pitch, (size_t)descs[i].out_width, (size_t)descs[i].out_height});
        if ((rc = l3d_stage_host(c, nullptr, 0, out.data(), n))) return rc;
    }
    s.h_imgs.assign(n, L3DJpegImage());
    s.h_tabs.resize((size_t)8 * n);
    s.h_segs.clear();
    size_t boff = 0;
    long long coef0 = 0, tile0 = 0;
    for (int i = 0; i < n; ++i) {
        const L3DJpegHeader& h = hdr[i];
        const l3d_jpeg_desc& u = descs[i];
        L3DJpegImage& d = s.h_imgs[i];
        memset(&d, 0, sizeof(d));
        const int64_t first = h.segs.front().first, len = h.segs.back().second - first;
        L3D_CUDA(c, cudaMemcpyAsync((unsigned char*)s.d_bytes.p + boff, u.data + first, (size_t)len, cudaMemcpyHostToDevice, c->stream), "upload JPEG data");
        const int ri = h.restart ? h.restart : h.mcus;
        for (size_t k = 0; k < h.segs.size(); ++k) {
            L3DJpegSeg g;
            g.first = (long long)(boff + (h.segs[k].first - first)); g.end = (long long)(boff + (h.segs[k].second - first));
            g.image = i; g.mcu0 = (int)(k * ri); g.mcu1 = (int)std::min<long long>((long long)(k + 1) * ri, h.mcus); g.pad = 0;
            s.h_segs.push_back(g);
        }
        boff += (size_t)len;
        if (on_device) { d.dst = u.dst; d.dst_pitch = u.dst_pitch; }
        else { d.dst = (unsigned char*)out[i].dev; d.dst_pitch = h.out_width; }
        d.coef0 = coef0; coef0 += (long long)h.yblocks_x * h.yblocks_y;
        d.tile0 = tile0;
        d.width = h.width; d.height = h.height; d.blocks_x = (h.width + 7) / 8;
        tile0 += (long long)d.blocks_x * ((h.height + 7) / 8);
        d.yblocks_x = h.yblocks_x; d.ns = h.ns; d.y_in_scan = h.y_in_scan; d.mcus_x = h.mcus_x;
        for (int k = 0; k < 4; ++k) { d.bh[k] = h.bh[k]; d.bv[k] = h.bv[k]; }
        jp_orientation(d, h.orientation);
        memcpy(d.q, h.q, sizeof(d.q));
        for (int k = 0; k < 4; ++k) {
            if (k < h.ns) { jp_table(h.dc[k], s.h_tabs[8 * i + 2 * k]); jp_table(h.ac[k], s.h_tabs[8 * i + 2 * k + 1]); }
            else { memset(&s.h_tabs[8 * i + 2 * k], 0, 2 * sizeof(L3DJpegTable)); }
        }
    }
    L3D_RESERVE(s.d_imgs, sizeof(L3DJpegImage) * (size_t)n, "JPEG image descriptors");
    L3D_RESERVE(s.d_segs, sizeof(L3DJpegSeg) * nseg, "JPEG segment descriptors");
    L3D_RESERVE(s.d_tabs, sizeof(L3DJpegTable) * s.h_tabs.size(), "JPEG Huffman tables");
    // pageable host memory: every copy is staged before it returns, so the host vectors may change right after
    L3D_CUDA(c, cudaMemcpyAsync(s.d_imgs.p, s.h_imgs.data(), sizeof(L3DJpegImage) * n, cudaMemcpyHostToDevice, c->stream), "upload JPEG descriptors");
    L3D_CUDA(c, cudaMemcpyAsync(s.d_segs.p, s.h_segs.data(), sizeof(L3DJpegSeg) * nseg, cudaMemcpyHostToDevice, c->stream), "upload JPEG segments");
    L3D_CUDA(c, cudaMemcpyAsync(s.d_tabs.p, s.h_tabs.data(), sizeof(L3DJpegTable) * s.h_tabs.size(), cudaMemcpyHostToDevice, c->stream),
             "upload JPEG tables");
    L3D_CUDA(c, cudaMemsetAsync(s.d_status.p, 0, sizeof(int) * n, c->stream), "clear JPEG status");
    // segments per warp: one while that still leaves four warps per SM, up to 32 when there are many
    int per_warp = 32;
    while (per_warp > 1 && (long long)(nseg + per_warp - 1) / per_warp < 4ll * c->num_sms) per_warp /= 2;
    k_jpeg_entropy<<<(unsigned int)((nseg + per_warp - 1) / per_warp), 32, 0, c->stream>>>((const L3DJpegSeg*)s.d_segs.p, (int)nseg, per_warp,
        (const L3DJpegImage*)s.d_imgs.p, (const L3DJpegTable*)s.d_tabs.p, (const unsigned char*)s.d_bytes.p, (short*)s.d_coefs.p, (int*)s.d_status.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_jpeg_entropy");
    k_jpeg_idct<<<(unsigned int)((tiles + JP_IDCT_THREADS - 1) / JP_IDCT_THREADS), JP_IDCT_THREADS, 0, c->stream>>>((const L3DJpegImage*)s.d_imgs.p, n, tiles,
                                                                                                                (const short*)s.d_coefs.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_jpeg_idct");
    s.h_status.assign(n, 0);
    L3D_CUDA(c, cudaMemcpyAsync(s.h_status.data(), s.d_status.p, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream), "download JPEG status");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "l3d_decode_jpeg_gray_u8");
    for (int i = 0; i < n; ++i)
        if (s.h_status[i] != JP_OK) {
            const char* why = s.h_status[i] == JP_BAD_CODE ? "corrupt entropy-coded data (no Huffman code matches)"
                              : s.h_status[i] == JP_BAD_AC ? "corrupt entropy-coded data (AC coefficients past index 63)"
                                                           : "corrupt entropy-coded data (a segment ends early)";
            snprintf(buf, sizeof(buf), "l3d_decode_jpeg_gray_u8: image %d: %s", i, why);
            return l3d_fail(c, L3D_ERR_INVALID, buf);
        }
    if (!on_device && (rc = l3d_unstage_host(c, out.data(), n, "l3d_decode_jpeg_gray_u8"))) return rc;
    return L3D_OK;
}
