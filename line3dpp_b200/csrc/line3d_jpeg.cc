// line3d_jpeg.cc — the host side of JPEG decoding (DESIGN.md §4c): the marker parser behind l3d_jpeg_info and l3d_decode_jpeg_gray_u8,
// the file readers of include/line3d_io.h (readJPEGSize, readJPEGGray, readJPEGsGray) and their C wrappers.  Entropy decoding and the
// IDCT run on the GPU (l3d_jpeg.cu); nothing here touches the coded data beyond finding its segment boundaries.
//
// The subset is what libjpeg-turbo decodes to grey without colour conversion or upsampling: baseline and extended-sequential Huffman
// (SOF0 / SOF1), 8-bit, one or three components with Y at the largest sampling factors, interleaved or not, with or without restart
// intervals.  Everything else is rejected with a message that names the reason; so is corrupt data, which libjpeg would patch up.
#include "l3d_exif.h"
#include "l3d_image_files.h"
#include "l3d_jpeg.h"
#include "../../include/line3d_io.h"
#include "../../include/l3d_capi.h"
#include "../../include/l3dpp_capi.h"
#include "l3dpp_wrap.h"

#include <cstring>
#include <fstream>
#include <iterator>

// zig-zag position -> natural index
static const uint8_t kZigZag[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
                                    62, 63};

static bool fail(std::string& err, const std::string& msg) { err = msg; return false; }

// libjpeg's checks of a DHT table (jpeg_make_d_derived_tbl): no length overflows its code space; DC symbols are sizes up to 15
static bool huff_ok(const L3DJpegHuffSpec& t, int count, bool dc)
{
    long code = 0;
    for (int l = 1; l <= 16; ++l) {
        code += t.bits[l - 1];
        if (code >= (1l << l)) return false;
        code <<= 1;
    }
    for (int i = 0; dc && i < count; ++i)
        if (t.vals[i] > 15) return false;
    return true;
}

// the entropy-coded data from pos: segments split at RSTn (their numbers into rst), and the position of the 0xFF of the marker that
// ends the scan.  A 0xFF followed by fill bytes and 0x00 is a stuffed data byte; fill bytes before a marker belong to no segment.
static bool scan_segments(const uint8_t* d, int64_t n, int64_t pos, std::vector<std::pair<int64_t, int64_t> >& segs, std::vector<int>& rst,
                          int64_t& marker, std::string& err)
{
    int64_t start = pos, i = pos;
    for (;;) {
        const uint8_t* f = (const uint8_t*)memchr(d + i, 0xFF, (size_t)(n - i));
        if (!f) return fail(err, "truncated entropy-coded data");
        i = f - d;
        int64_t j = i + 1;
        while (j < n && d[j] == 0xFF) ++j;
        if (j >= n) return fail(err, "truncated entropy-coded data");
        if (d[j] == 0x00) { i = j + 1; continue; }
        segs.push_back(std::make_pair(start, i));
        if (d[j] >= 0xD0 && d[j] <= 0xD7) { rst.push_back(d[j] - 0xD0); start = i = j + 1; continue; }
        marker = i;
        return true;
    }
}

static const char* rejected(int m)
{
    switch (m) {
    case 0xC2: case 0xC6: case 0xCA: case 0xCE: return "progressive JPEG is not supported";
    case 0xC3: case 0xC7: case 0xCB: case 0xCF: return "lossless JPEG is not supported";
    case 0xC5: case 0xDE: case 0xDF: return "hierarchical JPEG is not supported";
    case 0xC9: case 0xCC: case 0xCD: return "arithmetic coding is not supported";
    case 0xDC: return "DNL markers are not supported";
    default: return nullptr;
    }
}

bool l3d_jpeg_parse(const uint8_t* d, int64_t n, L3DJpegHeader& h, std::string& err)
{
    h = L3DJpegHeader();
    if (!d || n < 2 || d[0] != 0xFF || d[1] != 0xD8) return fail(err, "not a JPEG file (no SOI marker)");
    struct Comp { int id, h, v, tq; bool scanned; };
    std::vector<Comp> comps;
    uint16_t q[4][64];
    bool have_q[4] = {false, false, false, false}, have_dc[4] = {false, false, false, false}, have_ac[4] = {false, false, false, false};
    L3DJpegHuffSpec dc[4], ac[4];
    int ri = 0, orient = 0, adobe = -1, hmax = 1, vmax = 1;
    bool jfif = false, exif_seen = false, sof = false, y_scanned = false;
    int64_t pos = 2;
    for (;;) {
        if (pos >= n) return fail(err, "missing EOI marker");
        if (d[pos] != 0xFF) return fail(err, "corrupt data between markers");
        while (pos < n && d[pos] == 0xFF) ++pos;
        if (pos >= n) return fail(err, "missing EOI marker");
        const int m = d[pos++];
        if (m == 0xD9) break;
        if (const char* why = rejected(m)) return fail(err, why);
        if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) {
            char buf[64];
            snprintf(buf, sizeof(buf), "unexpected marker 0x%02X", m);
            return fail(err, buf);
        }
        if (pos + 2 > n) return fail(err, "truncated marker segment");
        const int64_t len = d[pos] << 8 | d[pos + 1];
        if (len < 2 || pos + len > n) return fail(err, "truncated marker segment");
        const uint8_t* p = d + pos + 2;
        const int64_t pn = len - 2, seg_end = pos + len;
        pos = seg_end;
        if (m >= 0xE0 && m <= 0xEF) {
            if (m == 0xE0 && pn >= 14 && !memcmp(p, "JFIF\0", 5)) jfif = true;
            else if (m == 0xE1 && !exif_seen && pn >= 6 && !memcmp(p, "Exif\0\0", 6)) { exif_seen = true; orient = l3d_exif_orientation(p + 6, pn - 6); }
            else if (m == 0xEE && pn >= 12 && !memcmp(p, "Adobe", 5)) adobe = p[11];
        } else if (m == 0xFE) {
        } else if (m == 0xDB) {
            for (int64_t i = 0; i < pn;) {
                const int pq = p[i] >> 4, tq = p[i] & 15, sz = 64 * (pq + 1);
                if (pq > 1 || tq > 3 || i + 1 + sz > pn) return fail(err, "corrupt quantisation table");
                for (int k = 0; k < 64; ++k) q[tq][kZigZag[k]] = pq ? (uint16_t)(p[i + 1 + 2 * k] << 8 | p[i + 2 + 2 * k]) : p[i + 1 + k];
                have_q[tq] = true;
                i += 1 + sz;
            }
        } else if (m == 0xC4) {
            for (int64_t i = 0; i < pn;) {
                if (i + 17 > pn) return fail(err, "corrupt Huffman table");
                const int tc = p[i] >> 4, th = p[i] & 15;
                int cnt = 0;
                for (int l = 0; l < 16; ++l) cnt += p[i + 1 + l];
                if (tc > 1 || th > 3 || cnt > 256 || i + 17 + cnt > pn) return fail(err, "corrupt Huffman table");
                L3DJpegHuffSpec& t = tc == 0 ? dc[th] : ac[th];
                memset(&t, 0, sizeof(t));
                memcpy(t.bits, p + i + 1, 16);
                memcpy(t.vals, p + i + 17, cnt);
                if (!huff_ok(t, cnt, tc == 0)) return fail(err, "corrupt Huffman table");
                (tc == 0 ? have_dc : have_ac)[th] = true;
                i += 17 + cnt;
            }
        } else if (m == 0xDD) {
            if (len != 4) return fail(err, "corrupt DRI marker");
            ri = p[0] << 8 | p[1];
        } else if (m == 0xC0 || m == 0xC1) {
            if (sof) return fail(err, "more than one frame header");
            if (pn < 6) return fail(err, "corrupt frame header");
            const int prec = p[0], hh = p[1] << 8 | p[2], ww = p[3] << 8 | p[4], nc = p[5];
            if (prec != 8) return fail(err, std::to_string(prec) + "-bit precision is not supported");
            if (hh == 0) return fail(err, "DNL markers are not supported");
            if (nc != 1 && nc != 3) return fail(err, std::to_string(nc) + " components are not supported (only grey and YCbCr)");
            if (pn != 6 + 3 * nc) return fail(err, "corrupt frame header");
            if (ww < 1 || ww > 32767 || hh < 1 || hh > 32767) return fail(err, "image side outside [1, 32767]");
            for (int c = 0; c < nc; ++c) {
                const Comp k = {p[6 + 3 * c], p[7 + 3 * c] >> 4, p[7 + 3 * c] & 15, p[8 + 3 * c], false};
                if (k.h < 1 || k.h > 4 || k.v < 1 || k.v > 4 || k.tq > 3) return fail(err, "corrupt frame header");
                comps.push_back(k);
                hmax = std::max(hmax, k.h); vmax = std::max(vmax, k.v);
            }
            h.width = ww; h.height = hh; sof = true;
        } else if (m == 0xDA) {
            if (!sof) return fail(err, "scan before the frame header");
            const int ns = pn > 0 ? p[0] : 0;
            if (ns < 1 || ns > 4 || pn != 4 + 2 * ns) return fail(err, "corrupt scan header");
            if (p[1 + 2 * ns] != 0 || p[2 + 2 * ns] != 63 || p[3 + 2 * ns] != 0) return fail(err, "corrupt scan header");
            int ci[4], td[4], ta[4], blocks = 0;
            bool has_y = false;
            for (int k = 0; k < ns; ++k) {
                ci[k] = -1;
                for (size_t c = 0; c < comps.size(); ++c)
                    if (comps[c].id == p[1 + 2 * k]) { if (ci[k] >= 0) return fail(err, "corrupt scan header"); ci[k] = (int)c; }
                if (ci[k] < 0 || comps[ci[k]].scanned) return fail(err, "corrupt scan header");
                td[k] = p[2 + 2 * k] >> 4; ta[k] = p[2 + 2 * k] & 15;
                if (td[k] > 3 || ta[k] > 3 || !have_dc[td[k]] || !have_ac[ta[k]]) return fail(err, "missing Huffman table");
                if (!have_q[comps[ci[k]].tq]) return fail(err, "missing quantisation table");
                comps[ci[k]].scanned = true;
                blocks += comps[ci[k]].h * comps[ci[k]].v;
                if (ci[k] == 0) { has_y = true; h.y_in_scan = k; }
            }
            if (ns > 1 && blocks > 10) return fail(err, "corrupt scan header");
            // the scan's MCU grid: one block of the component's own grid per MCU when it is alone, else the frame's MCUs
            int mx, my;
            if (ns == 1) {
                const Comp& c = comps[ci[0]];
                mx = (int)((((int64_t)h.width * c.h + hmax - 1) / hmax + 7) / 8);
                my = (int)((((int64_t)h.height * c.v + vmax - 1) / vmax + 7) / 8);
            } else {
                mx = (h.width + 8 * hmax - 1) / (8 * hmax);
                my = (h.height + 8 * vmax - 1) / (8 * vmax);
            }
            std::vector<std::pair<int64_t, int64_t> > segs;
            std::vector<int> rst;
            if (!scan_segments(d, n, seg_end, segs, rst, pos, err)) return false;
            const int64_t mcus = (int64_t)mx * my, need = ri ? (mcus + ri - 1) / ri : 1;
            bool ok = (int64_t)segs.size() == need;
            for (size_t k = 0; ok && k < rst.size(); ++k) ok = rst[k] == (int)(k % 8);
            if (!ok) return fail(err, "corrupt restart markers");
            if (has_y) {
                h.ns = ns; h.mcus_x = mx; h.mcus = (int)mcus; h.restart = ri; h.segs.swap(segs);
                for (int k = 0; k < ns; ++k) {
                    h.bh[k] = ns > 1 ? comps[ci[k]].h : 1; h.bv[k] = ns > 1 ? comps[ci[k]].v : 1;
                    h.dc[k] = dc[td[k]]; h.ac[k] = ac[ta[k]];
                }
                memcpy(h.q, q[comps[0].tq], sizeof(h.q));
                h.yblocks_x = mx * h.bh[h.y_in_scan]; h.yblocks_y = my * h.bv[h.y_in_scan];
                y_scanned = true;
            }
        } else {
            char buf[64];
            snprintf(buf, sizeof(buf), "unexpected marker 0x%02X", m);
            return fail(err, buf);
        }
    }
    if (!sof) return fail(err, "no frame header");
    for (const Comp& c : comps)
        if (!c.scanned) return fail(err, "a component has no scan");
    if (!y_scanned) return fail(err, "a component has no scan");
    // libjpeg's guess of the colour space of a 3-component file (jdapimin.c default_decompress_parms): RGB is not decoded here
    if (comps.size() == 3 && !jfif && (adobe == 0 || (adobe < 0 && comps[0].id == 'R' && comps[1].id == 'G' && comps[2].id == 'B')))
        return fail(err, "RGB JPEG is not supported");
    if (comps[0].h != hmax || comps[0].v != vmax) return fail(err, "Y is not at the largest sampling factors (it would need upsampling)");
    h.orientation = orient >= 1 && orient <= 8 ? orient : 1;
    h.out_width = h.orientation >= 5 ? h.height : h.width;
    h.out_height = h.orientation >= 5 ? h.width : h.height;
    return true;
}

extern "C" int l3d_jpeg_info(const uint8_t* data, int64_t size, int32_t* out_width, int32_t* out_height)
{
    if (!data || size < 0 || !out_width || !out_height) return L3D_ERR_INVALID;
    L3DJpegHeader h;
    std::string err;
    if (!l3d_jpeg_parse(data, size, h, err)) return L3D_ERR_INVALID;
    *out_width = h.out_width; *out_height = h.out_height;
    return L3D_OK;
}

// ------------------------------------------------------------------------------------------------ files
namespace L3DPP {

bool readJPEGSize(const std::string& path, int& width, int& height, std::string* error)
{
    std::vector<uint8_t> bytes;
    std::string err;
    L3DJpegHeader h;
    if (!l3d_read_file(path, bytes, err) || (!l3d_jpeg_parse(bytes.data(), (int64_t)bytes.size(), h, err) && (err = path + ": " + err, true))) {
        if (error) *error = err;
        return false;
    }
    width = h.out_width; height = h.out_height;
    return true;
}

bool readJPEGsGray(const std::vector<std::string>& paths, std::vector<Image8u>& images, std::vector<std::string>* errors, int cuda_device)
{
    auto parse = [](const uint8_t* d, int64_t n, int& w, int& h, std::string& err) {
        L3DJpegHeader hd;
        if (!l3d_jpeg_parse(d, n, hd, err)) return false;
        w = hd.out_width; h = hd.out_height;
        return true;
    };
    return l3d_read_gray_files<l3d_jpeg_desc>(paths, images, errors, cuda_device, parse, l3d_decode_jpeg_gray_u8, "JPEG");
}

bool readJPEGGray(const std::string& path, Image8u& image, std::string* error, int cuda_device)
{
    std::vector<Image8u> images;
    std::vector<std::string> errors;
    const bool ok = readJPEGsGray(std::vector<std::string>(1, path), images, &errors, cuda_device);
    image = images[0];
    if (!ok && error) *error = errors[0];
    return ok;
}

}  // namespace L3DPP

// C wrappers (include/l3dpp_capi.h): a batch of decoded files is a handle
extern "C" {
int l3dpp_jpeg_size(const char* path, int* width, int* height, char* err, int errcap)
{
    std::string e;
    if (!L3DPP::readJPEGSize(path, *width, *height, &e)) { l3dpp_copy_str(e, err, errcap); return -1; }
    return 0;
}

void* l3dpp_jpegs_read(const char* const* paths, int n, int cuda_device)
{
    L3DImageBatch* b = new L3DImageBatch();
    L3DPP::readJPEGsGray(std::vector<std::string>(paths, paths + (n > 0 ? n : 0)), b->images, &b->errors, cuda_device);
    return b;
}

void l3dpp_jpegs_close(void* h) { delete (L3DImageBatch*)h; }

int l3dpp_jpegs_image(void* h, int i, int* width, int* height, unsigned char* out, long long cap, char* err, int errcap)
{
    return l3d_batch_image(h, i, width, height, out, cap, err, errcap);
}
}
