// l3d_png.cu — imread(path, IMREAD_GRAYSCALE) of a batch of PNG files on the GPU, and its C-ABI entry point l3d_decode_png_gray_u8
// (include/l3d_capi.h).  The host parses the chunks (line3d_png.cc); three kernels do the rest, each one launch for the whole batch:
//   k_png_inflate   one warp per image: the zlib stream of its IDAT payload into the filtered rows of every pass.  The bit reader
//                   is warp-uniform (every lane decodes the same symbol); lanes store literals in 32-byte bursts and copy a match's
//                   bytes together.  Huffman tables are built in shared memory per block of data.  Every length, distance and
//                   write is checked against the bytes produced so far and the raw size; violations are a status, never a fault.
//   k_png_unfilter  filters 0..4 undone in place: per Adam7 pass, warps take bands of 32 rows, lane r a row, each row one unit
//                   (bpp bytes) behind the row above (a diagonal wavefront, __syncwarp between steps); a band waits for the band
//                   above it through a progress word in shared memory.
//   k_png_gray      one thread per output pixel: the EXIF orientation and Adam7 back to the sample, bit unpacking, the palette and
//                   libpng's grey rule with its gamma tables; each pixel stored once.
// The arithmetic contract is DESIGN.md §4d; tests/png_model.py restates it.  Not a pipeline stage: only PngState's buffers and, in
// host mode, the context's staging pair change.
#include "l3d_ctx.cuh"
#include "l3d_exif.h"
#include "l3d_png.h"

#include <climits>
#include <cstdio>
#include <cstring>

#define PN_GRAY_THREADS 256
#define PN_UNFILTER_WARPS 16

// status of an image after the kernels (PngState::h_status); the largest code found is reported
#define PN_OK 0
#define PN_BAD_BLOCK 1        // block type 3
#define PN_BAD_STORED 2       // a stored block's LEN and NLEN disagree
#define PN_BAD_CODES 3        // an over-subscribed or incomplete code-length set, or a bad repeat in it
#define PN_BAD_SYMBOL 4       // no code matches, or a literal/length symbol 286/287 or distance symbol 30/31
#define PN_BAD_DIST 5         // a distance past the start of the output or beyond the zlib window
#define PN_OVERLONG 6         // the stream inflates to more bytes than the image holds
#define PN_SHORT 7            // the input ends inside the stream
#define PN_UNDERLONG 8        // the stream ends before the image is complete
#define PN_TRAILING 9         // bytes after the zlib stream
#define PN_ADLER 10           // the Adler-32 does not match
#define PN_BAD_FILTER 11      // a row's filter type is not 0..4

__constant__ unsigned short c_pn_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ unsigned char c_pn_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ unsigned short c_pn_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
                                                  6145, 8193, 12289, 16385, 24577};
__constant__ unsigned char c_pn_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ unsigned char c_pn_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// ------------------------------------------------------------------------------------------------ inflate
// LSB-first bit reader over one zlib stream, the same state in every lane.  Past the end it reads zero bytes and counts them in pad.
struct PnBits {
    const unsigned char* p;
    const unsigned char* end;
    unsigned long long buf;
    int n, pad;

    __device__ __forceinline__ void fill()
    {
        while (n <= 56) {
            unsigned int b = 0;
            if (p < end) b = __ldg(p++);
            else pad += 8;
            buf |= (unsigned long long)b << n;
            n += 8;
        }
    }
    __device__ __forceinline__ unsigned int bits(int k) const { return (unsigned int)(buf & ((1ull << k) - 1)); }
    __device__ __forceinline__ void skip(int k) { buf >>= k; n -= k; }
};

#define PN_LOOK 9
// a Huffman table in shared memory: a 9-bit lookahead (length << 9 | symbol; 0: a longer code or none), then the canonical decode
// of zlib's puff over the per-length counts and the symbols sorted by code
struct PnTable {
    unsigned short look[1 << PN_LOOK];
    unsigned short count[16];
    unsigned short sym[288];
};

// the table of lengths[0..n) (warp-cooperative); false (warp-uniform) for a set zlib rejects: over-subscribed, or incomplete unless
// allow_single and the set is one code of length 1 or no code at all (literal/length and distance codes of a dynamic block)
__device__ bool pn_build(PnTable& t, const unsigned char* lengths, int n, bool allow_single, unsigned short* codes)
{
    const int lane = threadIdx.x & 31;
    __shared__ int s_ok[1];
    if (lane == 0) {
        for (int l = 0; l < 16; ++l) t.count[l] = 0;
        for (int s = 0; s < n; ++s) ++t.count[lengths[s]];
        int left = 1, ok = 1, maxl = 0;
        for (int l = 1; l < 16; ++l) {
            left <<= 1;
            left -= t.count[l];
            if (left < 0) ok = 0;
            if (t.count[l]) maxl = l;
        }
        if (ok && left > 0 && !(allow_single && maxl == 1 && t.count[1] == 1) && !(allow_single && maxl == 0)) ok = 0;
        unsigned short offs[16], next[16];
        offs[1] = 0;
        for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + t.count[l];
        int code = 0;
        t.count[0] = 0;
        for (int l = 1; l < 16; ++l) { code = (code + t.count[l - 1]) << 1; next[l] = (unsigned short)code; }
        for (int s = 0; s < n; ++s)
            if (lengths[s]) { t.sym[offs[lengths[s]]++] = (unsigned short)s; codes[s] = next[lengths[s]]++; }
        s_ok[0] = ok;
    }
    for (int e = lane; e < (1 << PN_LOOK); e += 32) t.look[e] = 0;
    __syncwarp();
    const bool ok = s_ok[0] != 0;
    if (ok)
        for (int s = lane; s < n; s += 32) {
            const int l = lengths[s];
            if (l == 0 || l > PN_LOOK) continue;
            const unsigned int r = __brev((unsigned int)codes[s]) >> (32 - l);
            for (unsigned int e = r; e < (1u << PN_LOOK); e += 1u << l) t.look[e] = (unsigned short)(l << 9 | s);
        }
    __syncwarp();
    return ok;
}

// the next symbol, -1 if no code matches; needs 15 bits in the reader
__device__ __forceinline__ int pn_symbol(PnBits& b, const PnTable& t)
{
    const unsigned int e = t.look[b.bits(PN_LOOK)];
    if (e) { b.skip(e >> 9); return e & 511; }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        code |= (int)((b.buf >> (l - 1)) & 1);
        const int count = t.count[l];
        if (code - count < first) { b.skip(l); return t.sym[index + (code - first)]; }
        index += count;
        first = (first + count) << 1;
        code <<= 1;
    }
    return -1;
}

// Adler-32 of out[0, n) (warp-cooperative; the result in every lane)
__device__ unsigned int pn_adler(const unsigned char* out, long long n)
{
    const int lane = threadIdx.x & 31;
    unsigned long long s1 = 0, s2 = 0;
    unsigned int w = (unsigned int)((n - lane) % 65521);    // byte i weighs n - i in the second sum
    long long k = 0;
    for (long long i = lane; i < n; i += 32, ++k) {
        const unsigned int v = out[i];
        s1 += v;
        s2 += (unsigned long long)(v * w);
        w = w >= 32 ? w - 32 : w + 65521 - 32;
        if ((k & 4095) == 4095) { s1 %= 65521; s2 %= 65521; }
    }
    s1 %= 65521; s2 %= 65521;
    for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    const unsigned long long a = (1 + s1) % 65521, bsum = (s2 + (unsigned long long)(n % 65521)) % 65521;
    return (unsigned int)(bsum << 16 | a);
}

// One warp (one CTA) per image.  Output bytes are written with plain stores and read back with plain loads after __syncwarp, which
// orders the warp's own global writes; never through the read-only cache.
__global__ void __launch_bounds__(32) k_png_inflate(const L3DPngImage* __restrict__ imgs, const unsigned char* __restrict__ in, unsigned char* raw,
                                                    int* __restrict__ status)
{
    __shared__ PnTable s_lit, s_dist;
    __shared__ unsigned char s_len[320];
    __shared__ unsigned short s_codes[320];
    const int lane = threadIdx.x;
    const L3DPngImage* im = imgs + blockIdx.x;
    unsigned char* out = raw + im->raw0;
    const long long size = im->raw_size;
    const int window = im->window;
    PnBits b;
    b.p = in + im->in0 + 2; b.end = in + im->in0 + im->in_len; b.buf = 0; b.n = 0; b.pad = 0;
    long long pos = 0;
    int err = PN_OK, last = 0, look = 0;     // look: bits a failed code lookup examined without consuming them
    unsigned int lit = 0;    // lane k holds the k-th buffered literal
    int nlit = 0;
    while (!last && err == PN_OK) {
        b.fill();
        last = b.bits(1);
        const int type = b.bits(3) >> 1;
        b.skip(3);
        if (type == 3) { err = PN_BAD_BLOCK; break; }
        if (type == 0) {
            // stored: drop to a byte boundary, hand the buffered whole bytes back to the input, then copy LEN bytes
            b.skip(b.n & 7);
            if (b.n < b.pad) { err = PN_SHORT; break; }
            b.p -= (b.n - b.pad) >> 3;
            b.buf = 0; b.n = 0; b.pad = 0;
            if (b.end - b.p < 4) { err = PN_SHORT; break; }
            const int len = __ldg(b.p) | __ldg(b.p + 1) << 8, nlen = __ldg(b.p + 2) | __ldg(b.p + 3) << 8;
            b.p += 4;
            if ((len ^ 0xFFFF) != nlen) { err = PN_BAD_STORED; break; }
            if (b.end - b.p < len) { err = PN_SHORT; break; }
            if (pos + len > size) { err = PN_OVERLONG; break; }
            for (int i = lane; i < len; i += 32) out[pos + i] = __ldg(b.p + i);
            b.p += len;
            pos += len;
            __syncwarp();
            continue;
        }
        // the block's codes
        if (type == 1) {
            for (int s = lane; s < 320; s += 32) s_len[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
            __syncwarp();
            // the fixed codes are complete: 288 literal/length codes, 32 distance codes of 5 bits (30 and 31 decode, and are invalid)
            if (!pn_build(s_lit, s_len, 288, false, s_codes) || !pn_build(s_dist, s_len + 288, 32, false, s_codes + 288)) { err = PN_BAD_CODES; break; }
        } else {
            const int nl = b.bits(5) + 257, nd = (b.bits(10) >> 5) + 1, nc = (b.bits(14) >> 10) + 4;
            b.skip(14);
            if (nl > 286 || nd > 30) { err = PN_BAD_CODES; break; }
            if (lane == 0)
                for (int s = 0; s < 19; ++s) s_len[s] = 0;
            __syncwarp();
            for (int k = 0; k < nc; ++k) {
                if (b.n < 3) b.fill();
                if (lane == 0) s_len[c_pn_cl_order[k]] = (unsigned char)b.bits(3);
                b.skip(3);
            }
            __syncwarp();
            if (!pn_build(s_dist, s_len, 19, false, s_codes)) { err = PN_BAD_CODES; break; }   // the code-length code, in s_dist for now
            __syncwarp();
            // the literal/length and distance lengths as one sequence (repeats may cross from one to the other), into s_len[0..nl + nd)
            unsigned char* lens = s_len;
            int k = 0, prev = -1;
            while (k < nl + nd) {
                if (b.n < 16) b.fill();
                const int s = pn_symbol(b, s_dist);
                if (s < 0) { err = PN_BAD_CODES; look = 15; break; }
                int rep, val;
                if (s < 16) { rep = 1; val = s; prev = s; }
                else if (s == 16) { if (prev < 0) { err = PN_BAD_CODES; break; } rep = 3 + b.bits(2); b.skip(2); val = prev; }
                else if (s == 17) { rep = 3 + b.bits(3); b.skip(3); val = 0; prev = 0; }
                else { rep = 11 + b.bits(7); b.skip(7); val = 0; prev = 0; }
                if (k + rep > nl + nd) { err = PN_BAD_CODES; break; }
                __syncwarp();
                for (int i = lane; i < rep; i += 32) lens[k + i] = (unsigned char)val;
                k += rep;
            }
            if (err != PN_OK) break;
            __syncwarp();
            if (lens[256] == 0) { err = PN_BAD_CODES; break; }
            // move the distance lengths to s_len[288..] (lanes read before anyone writes)
            unsigned char dl = lane < nd ? lens[nl + lane] : 0;
            __syncwarp();
            for (int s = nl + lane; s < 288; s += 32) lens[s] = 0;
            __syncwarp();
            if (lane < 30) lens[288 + lane] = dl;
            __syncwarp();
            if (!pn_build(s_lit, lens, 288, true, s_codes)) { err = PN_BAD_CODES; break; }
            if (!pn_build(s_dist, lens + 288, 30, true, s_codes + 288)) { err = PN_BAD_CODES; break; }
        }
        // the block's data
        for (;;) {
            if (b.n < 48) b.fill();
            const int s = pn_symbol(b, s_lit);
            if (s < 0 || s > 285) { err = PN_BAD_SYMBOL; look = s < 0 ? 15 : 0; break; }
            if (s < 256) {
                if (pos + nlit >= size) { err = PN_OVERLONG; break; }
                if (lane == nlit) lit = (unsigned int)s;
                if (++nlit == 32) { out[pos + lane] = (unsigned char)lit; pos += 32; nlit = 0; }
                continue;
            }
            if (nlit) { if (lane < nlit) out[pos + lane] = (unsigned char)lit; pos += nlit; nlit = 0; }
            if (s == 256) break;
            const int li = s - 257;
            const int len = c_pn_len_base[li] + (int)b.bits(c_pn_len_extra[li]);
            b.skip(c_pn_len_extra[li]);
            const int ds = pn_symbol(b, s_dist);
            if (ds < 0 || ds > 29) { err = PN_BAD_SYMBOL; look = ds < 0 ? 15 : 0; break; }
            const int dist = c_pn_dist_base[ds] + (int)b.bits(c_pn_dist_extra[ds]);
            b.skip(c_pn_dist_extra[ds]);
            if (dist > pos || dist > window) { err = PN_BAD_DIST; break; }
            if (pos + len > size) { err = PN_OVERLONG; break; }
            __syncwarp();
            // every byte of the copy comes from before pos: with an overlap (dist < len) the pattern repeats with period dist
            for (int i = lane; i < len; i += 32) out[pos + i] = out[pos - dist + (dist < len ? i % dist : i)];
            pos += len;
            __syncwarp();
        }
        if (err == PN_OK && b.n < b.pad) err = PN_SHORT;      // some of the zero bits read past the end were used
    }
    // an error found in bits that reach past the end of the input is the input ending early, whatever the padding decoded to
    if (err != PN_OK && b.n - look < b.pad) err = PN_SHORT;
    if (err == PN_OK && nlit) { if (lane < nlit) out[pos + lane] = (unsigned char)lit; pos += nlit; nlit = 0; }
    __syncwarp();
    if (err == PN_OK && pos != size) err = PN_UNDERLONG;
    if (err == PN_OK) {
        // the Adler-32 at the next byte boundary, then the end of the input
        b.skip(b.n & 7);
        if (b.n < b.pad) err = PN_SHORT;
        else {
            b.p -= (b.n - b.pad) >> 3;
            if (b.end - b.p < 4) err = PN_SHORT;
            else {
                const unsigned int want = (unsigned int)__ldg(b.p) << 24 | (unsigned int)__ldg(b.p + 1) << 16 | (unsigned int)__ldg(b.p + 2) << 8 | __ldg(b.p + 3);
                if (b.end - b.p > 4) err = PN_TRAILING;
                else if (pn_adler(out, size) != want) err = PN_ADLER;
            }
        }
    }
    if (err != PN_OK && lane == 0) atomicMax(status + blockIdx.x, err);
}

// ------------------------------------------------------------------------------------------------ unfilter
__device__ __forceinline__ int pn_paeth(int a, int b, int c)
{
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

// One CTA of PN_UNFILTER_WARPS warps per pass; warp w takes bands w, w + W, ... of 32 rows.  At step t lane r undoes unit t - r of
// its row (bpp bytes; units need row r-1's unit t-r, done at step t-1).  s_prog[w] = (band << 32 | units done in the band's last
// row) tells the warp of the next band how far it may go.
__global__ void __launch_bounds__(PN_UNFILTER_WARPS * 32) k_png_unfilter(const L3DPngPass* __restrict__ passes, unsigned char* raw,
                                                                        const L3DPngImage* __restrict__ imgs, int* __restrict__ status)
{
    __shared__ volatile long long s_prog[PN_UNFILTER_WARPS];
    const L3DPngPass ps = passes[blockIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned char* base = raw + imgs[ps.image].raw0 + ps.off;
    const int bpp = ps.bpp, rb = ps.rb, units = rb / bpp, rows = ps.rows;
    const long long stride = rb + 1;
    if (status[ps.image] != PN_OK) return;                 // the inflate failed: its reason is the one reported
    s_prog[warp] = -1;
    __syncthreads();
    int bad = 0;
    for (int band = warp; band * 32 < rows; band += PN_UNFILTER_WARPS) {
        const int y = band * 32 + lane;
        const bool live = y < rows;
        unsigned char* row = base + (long long)y * stride;
        const unsigned char* up = row - stride;
        int f = live ? row[0] : 0;
        if (f > 4) { bad = 1; f = 0; }
        const int pw = (warp + PN_UNFILTER_WARPS - 1) % PN_UNFILTER_WARPS;
        unsigned int a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, c[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int t = 0; t < units + 31; ++t) {
            const int x = t - lane;
            // lane 0 needs unit x of the band above's last row
            if (band > 0 && lane == 0 && x >= 0 && x < units) {
                const long long need = (long long)(band - 1) << 32 | (unsigned int)(x + 1);
                while (s_prog[pw] < need) {}
                __threadfence_block();
            }
            __syncwarp();
            if (live && x >= 0 && x < units) {
                unsigned char* q = row + 1 + (long long)x * bpp;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (k >= bpp) break;
                    const unsigned int bb = y > 0 ? up[1 + (long long)x * bpp + k] : 0;
                    const unsigned int v = q[k];
                    unsigned int r;
                    switch (f) {
                    case 1: r = v + a[k]; break;
                    case 2: r = v + bb; break;
                    case 3: r = v + ((a[k] + bb) >> 1); break;
                    case 4: r = v + (unsigned int)pn_paeth((int)a[k], (int)bb, (int)c[k]); break;
                    default: r = v; break;
                    }
                    r &= 255;
                    q[k] = (unsigned char)r;
                    a[k] = r; c[k] = bb;
                }
            }
            __syncwarp();
            if (lane == 31 && live && x >= 0 && x < units) {
                __threadfence_block();
                s_prog[warp] = (long long)band << 32 | (unsigned int)(x + 1);
            }
        }
    }
    if (bad) atomicMax(status + ps.image, PN_BAD_FILTER);
}

// ------------------------------------------------------------------------------------------------ grey conversion
__constant__ unsigned char c_pn_adam7_pass[64] = {0, 5, 3, 5, 1, 5, 3, 5, 6, 6, 6, 6, 6, 6, 6, 6, 4, 5, 4, 5, 4, 5, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6,
                                                  2, 5, 3, 5, 2, 5, 3, 5, 6, 6, 6, 6, 6, 6, 6, 6, 4, 5, 4, 5, 4, 5, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6};
__constant__ unsigned char c_pn_adam7[7][4] = {{0, 0, 8, 8}, {4, 0, 8, 8}, {0, 4, 4, 8}, {2, 0, 4, 4}, {0, 2, 2, 4}, {1, 0, 2, 2}, {0, 1, 1, 2}};

// sample k of unit x of a row (depth 1, 2, 4, 8 or 16; 16-bit samples whole)
__device__ __forceinline__ unsigned int pn_sample(const unsigned char* row, int x, int k, int ch, int depth)
{
    if (depth == 8) return row[(long long)x * ch + k];
    if (depth == 16) { const long long o = 2 * ((long long)x * ch + k); return (unsigned int)row[o] << 8 | row[o + 1]; }
    const long long bit = (long long)x * depth;
    return (row[bit >> 3] >> (8 - depth - (int)(bit & 7))) & ((1u << depth) - 1);
}

__global__ void __launch_bounds__(PN_GRAY_THREADS) k_png_gray(const L3DPngImage* __restrict__ imgs, int n, long long total, const unsigned char* __restrict__ raw)
{
    const long long t = (long long)blockIdx.x * PN_GRAY_THREADS + threadIdx.x;
    if (t >= total) return;
    const L3DPngImage* im = imgs + last_le(n, t, [&](int i) { return imgs[i].pix0; });
    const long long local = t - im->pix0;
    const int r = (int)(local / im->out_width), cc = (int)(local % im->out_width);
    // the inverse of the orientation map (its linear part is orthogonal): the coded pixel (y, x)
    const int dr = r - im->ry0, dc = cc - im->rx0;
    const int y = im->ryy * dr + im->rxy * dc, x = im->ryx * dr + im->rxx * dc;
    int pass = 0, py = y, px = x;
    if (im->interlace) {
        pass = c_pn_adam7_pass[(y & 7) * 8 + (x & 7)];
        py = (y - c_pn_adam7[pass][1]) / c_pn_adam7[pass][3];
        px = (x - c_pn_adam7[pass][0]) / c_pn_adam7[pass][2];
    }
    const unsigned char* row = raw + im->raw0 + im->pass_off[pass] + (long long)py * (im->pass_rb[pass] + 1) + 1;
    const int ct = im->color_type, depth = im->depth, ch = im->channels;
    unsigned int g;
    if (ct == 0 || ct == 4) {
        const unsigned int v = pn_sample(row, px, 0, ch, depth);
        g = depth == 16 ? v >> 8 : depth == 8 ? v : v * (255u / ((1u << depth) - 1));
    } else {
        unsigned int R, G, B;
        if (ct == 3) {
            const unsigned int i = pn_sample(row, px, 0, 1, depth);
            R = __ldg(&im->palette[3 * i]); G = __ldg(&im->palette[3 * i + 1]); B = __ldg(&im->palette[3 * i + 2]);
        } else {
            R = pn_sample(row, px, 0, ch, depth); G = pn_sample(row, px, 1, ch, depth); B = pn_sample(row, px, 2, ch, depth);
        }
        if (R == G && R == B) g = depth == 16 ? R >> 8 : R;
        else if (depth == 16) g = ((9797u * R + 19234u * G + 3737u * B + 16384u) >> 15) >> 8;
        else if (im->gamma)
            g = __ldg(&im->from_linear[(9797u * __ldg(&im->to_linear[R]) + 19234u * __ldg(&im->to_linear[G]) + 3737u * __ldg(&im->to_linear[B]) + 16384u) >> 15]);
        else g = (9797u * R + 19234u * G + 3737u * B) >> 15;
    }
    im->dst[(long long)r * im->dst_pitch + cc] = (unsigned char)g;
}

// ------------------------------------------------------------------------------------------------ host side
static const char* pn_reason(int s)
{
    switch (s) {
    case PN_BAD_BLOCK: return "corrupt deflate stream (invalid block type)";
    case PN_BAD_STORED: return "corrupt deflate stream (stored block length does not match its complement)";
    case PN_BAD_CODES: return "corrupt deflate stream (bad code lengths)";
    case PN_BAD_SYMBOL: return "corrupt deflate stream (invalid code)";
    case PN_BAD_DIST: return "corrupt deflate stream (distance too far back)";
    case PN_OVERLONG: return "corrupt deflate stream (more data than the image holds)";
    case PN_SHORT: return "corrupt deflate stream (it ends early)";
    case PN_UNDERLONG: return "corrupt deflate stream (less data than the image holds)";
    case PN_TRAILING: return "data after the zlib stream";
    case PN_ADLER: return "corrupt deflate stream (Adler-32 mismatch)";
    default: return "corrupt image data (bad filter type)";
    }
}

extern "C" int l3d_decode_png_gray_u8(l3d_ctx* c, int n, const l3d_png_desc* descs, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    if (n < 0 || (n && !descs)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_decode_png_gray_u8: bad arguments");
    // every descriptor is checked (and every file parsed) before anything is launched
    std::vector<L3DPngHeader> hdr(n);
    char buf[512];
    for (int i = 0; i < n; ++i) {
        const l3d_png_desc& u = descs[i];
        std::string err;
        if (!u.data || u.size <= 0) err = "no file data";
        else if (!l3d_png_parse(u.data, u.size, hdr[i], err)) {}
        else if (!u.dst) err = "null dst";
        else if (u.out_width != hdr[i].out_width || u.out_height != hdr[i].out_height) {
            snprintf(buf, sizeof(buf), "out size %dx%d, but l3d_png_info gives %dx%d", u.out_width, u.out_height, hdr[i].out_width, hdr[i].out_height);
            err = buf;
        } else if (u.dst_pitch < u.out_width) err = "dst pitch below out_width";
        if (!err.empty()) {
            snprintf(buf, sizeof(buf), "l3d_decode_png_gray_u8: image %d: %s", i, err.c_str());
            return l3d_fail(c, L3D_ERR_INVALID, buf);
        }
    }
    if (n == 0) return L3D_OK;
    cudaSetDevice(c->device);
    PngState& s = c->png;
    int rc;
    size_t in_bytes = 0, raw_bytes = 0;
    long long pixels = 0;
    for (int i = 0; i < n; ++i) {
        in_bytes += (size_t)hdr[i].zlib_size;
        raw_bytes += ((size_t)hdr[i].raw_size + 15) & ~(size_t)15;
        pixels += (long long)hdr[i].width * hdr[i].height;
    }
    if (n > INT_MAX / 7 || (pixels + PN_GRAY_THREADS - 1) / PN_GRAY_THREADS >= (1ll << 31))
        return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_decode_png_gray_u8: too many pixels in one call");
    L3D_RESERVE(s.d_in, in_bytes, "PNG data staging");
    L3D_RESERVE(s.d_raw, raw_bytes, "PNG scanlines");
    L3D_RESERVE(s.d_status, sizeof(int) * (size_t)n, "PNG status");
    std::vector<HostBlock> out;             // host mode: every output
    if (!on_device) {
        for (int i = 0; i < n; ++i) out.push_back({descs[i].dst, (size_t)descs[i].dst_pitch, (size_t)descs[i].out_width, (size_t)descs[i].out_height});
        if ((rc = l3d_stage_host(c, nullptr, 0, out.data(), n))) return rc;
    }
    s.h_imgs.assign(n, L3DPngImage());
    s.h_passes.clear();
    s.h_in.resize(in_bytes);
    size_t ioff = 0, roff = 0;
    long long pix0 = 0;
    for (int i = 0; i < n; ++i) {
        const L3DPngHeader& h = hdr[i];
        L3DPngImage& d = s.h_imgs[i];
        memset(&d, 0, sizeof(d));
        d.in0 = (long long)ioff;
        for (const auto& r : h.idat) { memcpy(s.h_in.data() + ioff, descs[i].data + r.first, (size_t)(r.second - r.first)); ioff += (size_t)(r.second - r.first); }
        d.in_len = h.zlib_size;
        d.raw0 = (long long)roff; d.raw_size = h.raw_size;
        roff += ((size_t)h.raw_size + 15) & ~(size_t)15;
        d.pix0 = pix0; pix0 += (long long)h.width * h.height;
        if (on_device) { d.dst = descs[i].dst; d.dst_pitch = descs[i].dst_pitch; }
        else { d.dst = (unsigned char*)out[i].dev; d.dst_pitch = h.out_width; }
        for (int k = 0; k < 7; ++k) { d.pass_off[k] = h.pass_off[k]; d.pass_rb[k] = h.pass_rb[k]; }
        d.width = h.width; d.height = h.height; d.depth = h.depth; d.color_type = h.color_type; d.channels = h.channels; d.interlace = h.interlace;
        d.window = 1 << h.window_bits;
        d.out_width = h.out_width; d.out_height = h.out_height;
        d.gamma = h.gamma;
        int a[6];
        l3d_orientation_map(h.orientation, h.width, h.height, a);
        d.ryy = a[0]; d.ryx = a[1]; d.ry0 = a[2]; d.rxy = a[3]; d.rxx = a[4]; d.rx0 = a[5];
        memcpy(d.palette, h.palette, sizeof(d.palette));
        memcpy(d.to_linear, h.to_linear, sizeof(d.to_linear));
        memcpy(d.from_linear, h.from_linear, sizeof(d.from_linear));
        const int bpp = std::max(1, h.channels * h.depth / 8);
        for (int k = 0; k < (h.interlace ? 7 : 1); ++k)
            if (h.pass_w[k] && h.pass_h[k]) s.h_passes.push_back(L3DPngPass{h.pass_off[k], i, h.pass_h[k], (int)h.pass_rb[k], bpp});
    }
    L3D_RESERVE(s.d_imgs, sizeof(L3DPngImage) * (size_t)n, "PNG image descriptors");
    L3D_RESERVE(s.d_passes, sizeof(L3DPngPass) * s.h_passes.size(), "PNG passes");
    // pageable host memory: every copy is staged before it returns, so the host vectors may change right after
    L3D_CUDA(c, cudaMemcpyAsync(s.d_in.p, s.h_in.data(), in_bytes, cudaMemcpyHostToDevice, c->stream), "upload PNG data");
    L3D_CUDA(c, cudaMemcpyAsync(s.d_imgs.p, s.h_imgs.data(), sizeof(L3DPngImage) * n, cudaMemcpyHostToDevice, c->stream), "upload PNG descriptors");
    L3D_CUDA(c, cudaMemcpyAsync(s.d_passes.p, s.h_passes.data(), sizeof(L3DPngPass) * s.h_passes.size(), cudaMemcpyHostToDevice, c->stream), "upload PNG passes");
    L3D_CUDA(c, cudaMemsetAsync(s.d_status.p, 0, sizeof(int) * n, c->stream), "clear PNG status");
    k_png_inflate<<<n, 32, 0, c->stream>>>((const L3DPngImage*)s.d_imgs.p, (const unsigned char*)s.d_in.p, (unsigned char*)s.d_raw.p, (int*)s.d_status.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_png_inflate");
    k_png_unfilter<<<(unsigned int)s.h_passes.size(), PN_UNFILTER_WARPS * 32, 0, c->stream>>>((const L3DPngPass*)s.d_passes.p, (unsigned char*)s.d_raw.p,
                                                                                           (const L3DPngImage*)s.d_imgs.p, (int*)s.d_status.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_png_unfilter");
    k_png_gray<<<(unsigned int)((pixels + PN_GRAY_THREADS - 1) / PN_GRAY_THREADS), PN_GRAY_THREADS, 0, c->stream>>>((const L3DPngImage*)s.d_imgs.p, n, pixels,
                                                                                                                (const unsigned char*)s.d_raw.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_png_gray");
    s.h_status.assign(n, 0);
    L3D_CUDA(c, cudaMemcpyAsync(s.h_status.data(), s.d_status.p, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream), "download PNG status");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "l3d_decode_png_gray_u8");
    for (int i = 0; i < n; ++i)
        if (s.h_status[i] != PN_OK) {
            snprintf(buf, sizeof(buf), "l3d_decode_png_gray_u8: image %d: %s", i, pn_reason(s.h_status[i]));
            return l3d_fail(c, L3D_ERR_INVALID, buf);
        }
    if (!on_device && (rc = l3d_unstage_host(c, out.data(), n, "l3d_decode_png_gray_u8"))) return rc;
    return L3D_OK;
}
