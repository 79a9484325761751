// line3d_png.cc — the host side of PNG decoding (DESIGN.md §4d): the chunk parser behind l3d_png_info and l3d_decode_png_gray_u8,
// the file readers of include/line3d_io.h (readPNGSize, readPNGGray, readPNGsGray, and readImageSize / readImageGray /
// readImagesGray, which pick the JPEG or the PNG reader by the file's signature) and their C wrappers.  Inflating, unfiltering and
// the grey conversion run on the GPU (l3d_png.cu); nothing here touches the zlib stream beyond its two header bytes.
//
// The subset is every colour type and bit depth of PNG 1.2, interlaced or not, with OpenCV's grey conversion including libpng's gamma
// tables for gAMA / sRGB colour files of 8 bits or less.  Everything else is rejected with a message that names the reason; so is
// data that libpng would only warn about (a bad ancillary CRC, extra compressed data, chunks out of place).
#include "l3d_exif.h"
#include "l3d_image_files.h"
#include "l3d_png.h"
#include "../../include/line3d_io.h"
#include "../../include/l3d_capi.h"
#include "../../include/l3dpp_capi.h"
#include "l3dpp_wrap.h"

#include <cmath>
#include <cstring>
#include <fstream>
#include <iterator>

static bool fail(std::string& err, const std::string& msg) { err = msg; return false; }

static uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

static uint32_t crc32_png(const uint8_t* p, int64_t n)
{
    static uint32_t table[256];
    static bool init = false;
    if (!init) {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            table[i] = c;
        }
        init = true;
    }
    uint32_t c = 0xFFFFFFFFu;
    for (int64_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 255] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

// libpng's png_reciprocal, png_gamma_significant and png_build_8bit_table (floating-point arithmetic), in its 1e5 fixed point
static int64_t png_reciprocal(int64_t a) { return (int64_t)std::floor(1e10 / (double)a + .5); }
static bool gamma_significant(int64_t g) { return g < 100000 - 5000 || g > 100000 + 5000; }
static void gamma_table(int64_t g, uint8_t* t)
{
    for (int v = 0; v < 256; ++v)
        t[v] = (uint8_t)(!gamma_significant(g) || v == 0 || v == 255 ? v : (int)std::floor(255 * std::pow(v / 255., (double)g * .00001) + .5));
}

static const int kAdam7[7][4] = {{0, 0, 8, 8}, {4, 0, 8, 8}, {0, 4, 4, 8}, {2, 0, 4, 4}, {0, 2, 2, 4}, {1, 0, 2, 2}, {0, 1, 1, 2}};   // x0, y0, dx, dy

static bool legal_depth(int ct, int d)
{
    switch (ct) {
    case 0: return d == 1 || d == 2 || d == 4 || d == 8 || d == 16;
    case 3: return d == 1 || d == 2 || d == 4 || d == 8;
    case 2: case 4: case 6: return d == 8 || d == 16;
    default: return false;
    }
}

static bool is_type(const uint8_t* t, const char* name) { return !memcmp(t, name, 4); }

bool l3d_png_parse(const uint8_t* d, int64_t n, L3DPngHeader& h, std::string& err)
{
    static const uint8_t kSig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    h = L3DPngHeader();
    if (!d || n < 8 || memcmp(d, kSig, 8)) return fail(err, "not a PNG file (no PNG signature)");
    int64_t pos = 8;
    bool first = true, have_plte = false, seen_idat = false, ended_idat = false, exif_seen = false, srgb = false;
    int64_t gamma = 0;
    int orient = 1;
    for (;;) {
        if (pos + 8 > n) return fail(err, "truncated chunk");
        const uint32_t len = be32(d + pos);
        const uint8_t* t = d + pos + 4;
        if (len > 0x7FFFFFFFu || pos + 12 + (int64_t)len > n) return fail(err, "truncated chunk");
        const uint8_t* p = d + pos + 8;
        if (crc32_png(t, 4 + (int64_t)len) != be32(p + len)) return fail(err, std::string("bad CRC in chunk ") + std::string((const char*)t, 4));
        const int64_t body = pos + 8;
        pos += 12 + (int64_t)len;
        for (int k = 0; k < 4; ++k)
            if (!((t[k] >= 'A' && t[k] <= 'Z') || (t[k] >= 'a' && t[k] <= 'z'))) return fail(err, "bad chunk type");
        const bool ihdr = is_type(t, "IHDR");
        if (first != ihdr) return fail(err, "IHDR is not the first chunk");
        first = false;
        const bool idat = is_type(t, "IDAT");
        if (!idat && seen_idat) ended_idat = true;
        if (ihdr) {
            if (len != 13) return fail(err, "corrupt IHDR");
            const uint32_t w = be32(p), hh = be32(p + 4);
            const int depth = p[8], ct = p[9];
            if (!legal_depth(ct, depth)) return fail(err, "invalid colour type and bit depth");
            if (p[10] != 0 || p[11] != 0 || p[12] > 1) return fail(err, "invalid compression, filter or interlace method");
            if (w < 1 || hh < 1 || w > 1000000 || hh > 1000000 || (uint64_t)w * hh > (1ull << 30)) return fail(err, "image size outside the supported limits");
            h.width = (int)w; h.height = (int)hh; h.depth = depth; h.color_type = ct; h.interlace = p[12];
            h.channels = ct == 0 || ct == 3 ? 1 : ct == 2 ? 3 : ct == 4 ? 2 : 4;
        } else if (is_type(t, "PLTE")) {
            if (have_plte || seen_idat || len % 3 || len == 0 || len > 768) return fail(err, "corrupt PLTE");
            if (h.color_type == 0 || h.color_type == 4) return fail(err, "PLTE in a grey image");
            if (h.color_type == 3 && len / 3 > (1u << h.depth)) return fail(err, "PLTE longer than the bit depth allows");
            memcpy(h.palette, p, len);
            have_plte = true;
        } else if (idat) {
            if (ended_idat) return fail(err, "IDAT chunks are not consecutive");
            seen_idat = true;
            h.idat.push_back(std::make_pair(body, body + (int64_t)len));
            h.zlib_size += len;
        } else if (is_type(t, "IEND")) {
            break;
        } else if (is_type(t, "tRNS")) {
            if (seen_idat) return fail(err, "tRNS out of place");
        } else if (is_type(t, "gAMA")) {
            if (len != 4 || seen_idat || have_plte) return fail(err, "gAMA out of place or corrupt");
            if (gamma) return fail(err, "more than one gAMA");      // libpng keeps the first and warns
            gamma = be32(p);
            if (gamma < 16 || gamma > 625000000) return fail(err, "gAMA value out of range");
        } else if (is_type(t, "sRGB")) {
            if (len != 1 || seen_idat || have_plte) return fail(err, "sRGB out of place or corrupt");
            if (srgb) return fail(err, "more than one sRGB");
            if (p[0] > 3) return fail(err, "sRGB rendering intent out of range");   // libpng ignores such a chunk and warns
            srgb = true;
        } else if (is_type(t, "iCCP")) {
            return fail(err, "iCCP colour profiles are not supported");
        } else if (is_type(t, "cHRM")) {
            return fail(err, "cHRM chromaticities are not supported");
        } else if (is_type(t, "cICP")) {
            return fail(err, "cICP colour information is not supported");
        } else if (is_type(t, "acTL") || is_type(t, "fcTL") || is_type(t, "fdAT")) {
            return fail(err, "animated PNG is not supported");
        } else if (is_type(t, "eXIf")) {
            if (!exif_seen) { exif_seen = true; orient = l3d_exif_orientation(p, len); }
        } else if (!(t[0] & 32)) {
            return fail(err, std::string("unknown critical chunk ") + std::string((const char*)t, 4));
        }
    }
    if (pos != n) return fail(err, "data after IEND");
    if (h.idat.empty()) return fail(err, "no IDAT chunk");
    if (h.color_type == 3 && !have_plte) return fail(err, "palette image without PLTE");
    if (srgb && gamma && gamma != 45455) return fail(err, "gAMA and sRGB disagree");
    // libpng's rgb_to_gray with a file gamma and no screen gamma: the screen gamma is taken as the file gamma's reciprocal; tables are
    // built when either is significant (png_init_read_transformations)
    const int64_t fg = srgb ? 45455 : gamma;
    if (fg && (h.color_type & 2)) {
        const int64_t screen = png_reciprocal(fg);
        if (gamma_significant(fg) || gamma_significant(screen)) {
            if (h.depth == 16) return fail(err, "gamma correction of 16-bit colour is not supported");
            h.gamma = true;
            gamma_table(png_reciprocal(fg), h.to_linear);
            gamma_table(png_reciprocal(screen), h.from_linear);
        }
    }
    // the zlib header, which may be split over IDAT chunks
    uint8_t z[2];
    int got = 0;
    for (size_t k = 0; k < h.idat.size() && got < 2; ++k)
        for (int64_t i = h.idat[k].first; i < h.idat[k].second && got < 2; ++i) z[got++] = d[i];
    if (got < 2 || (z[0] & 15) != 8 || (z[0] >> 4) > 7 || (z[0] << 8 | z[1]) % 31) return fail(err, "corrupt zlib header");
    if (z[1] & 32) return fail(err, "zlib preset dictionary");
    h.window_bits = (z[0] >> 4) + 8;
    // the raw size: every pass with pixels, one filter byte per row
    const int np = h.interlace ? 7 : 1;
    int64_t off = 0;
    for (int k = 0; k < np; ++k) {
        const int x0 = h.interlace ? kAdam7[k][0] : 0, y0 = h.interlace ? kAdam7[k][1] : 0, dx = h.interlace ? kAdam7[k][2] : 1, dy = h.interlace ? kAdam7[k][3] : 1;
        h.pass_w[k] = h.width > x0 ? (h.width - x0 + dx - 1) / dx : 0;
        h.pass_h[k] = h.height > y0 ? (h.height - y0 + dy - 1) / dy : 0;
        h.pass_rb[k] = ((int64_t)h.pass_w[k] * h.channels * h.depth + 7) / 8;
        h.pass_off[k] = off;
        if (h.pass_w[k] && h.pass_h[k]) off += (int64_t)h.pass_h[k] * (h.pass_rb[k] + 1);
    }
    h.raw_size = off;
    h.orientation = orient >= 1 && orient <= 8 ? orient : 1;
    h.out_width = h.orientation >= 5 ? h.height : h.width;
    h.out_height = h.orientation >= 5 ? h.width : h.height;
    return true;
}

extern "C" int l3d_png_info(const uint8_t* data, int64_t size, int32_t* out_width, int32_t* out_height)
{
    if (!data || size < 0 || !out_width || !out_height) return L3D_ERR_INVALID;
    L3DPngHeader h;
    std::string err;
    if (!l3d_png_parse(data, size, h, err)) return L3D_ERR_INVALID;
    *out_width = h.out_width; *out_height = h.out_height;
    return L3D_OK;
}

// ------------------------------------------------------------------------------------------------ files
namespace L3DPP {

bool readPNGSize(const std::string& path, int& width, int& height, std::string* error)
{
    std::vector<uint8_t> bytes;
    std::string err;
    L3DPngHeader h;
    if (!l3d_read_file(path, bytes, err) || (!l3d_png_parse(bytes.data(), (int64_t)bytes.size(), h, err) && (err = path + ": " + err, true))) {
        if (error) *error = err;
        return false;
    }
    width = h.out_width; height = h.out_height;
    return true;
}

bool readPNGsGray(const std::vector<std::string>& paths, std::vector<Image8u>& images, std::vector<std::string>* errors, int cuda_device)
{
    auto parse = [](const uint8_t* d, int64_t n, int& w, int& h, std::string& err) {
        L3DPngHeader hd;
        if (!l3d_png_parse(d, n, hd, err)) return false;
        w = hd.out_width; h = hd.out_height;
        return true;
    };
    return l3d_read_gray_files<l3d_png_desc>(paths, images, errors, cuda_device, parse, l3d_decode_png_gray_u8, "PNG");
}

bool readPNGGray(const std::string& path, Image8u& image, std::string* error, int cuda_device)
{
    std::vector<Image8u> images;
    std::vector<std::string> errors;
    const bool ok = readPNGsGray(std::vector<std::string>(1, path), images, &errors, cuda_device);
    image = images[0];
    if (!ok && error) *error = errors[0];
    return ok;
}

// the reader a file's first bytes call for: 1 JPEG (SOI), 2 PNG (signature), 0 neither (err set)
static int image_kind(const std::string& path, std::string& err)
{
    std::ifstream f(path.c_str(), std::ios::binary);
    if (!f) { err = path + ": cannot open file"; return 0; }
    uint8_t b[8] = {};
    f.read((char*)b, 8);
    if (f.gcount() >= 2 && b[0] == 0xFF && b[1] == 0xD8) return 1;
    static const uint8_t kSig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    if (f.gcount() == 8 && !memcmp(b, kSig, 8)) return 2;
    err = path + ": not a JPEG or PNG file";
    return 0;
}

bool readImageSize(const std::string& path, int& width, int& height, std::string* error)
{
    std::string err;
    const int k = image_kind(path, err);
    if (k == 1) return readJPEGSize(path, width, height, error);
    if (k == 2) return readPNGSize(path, width, height, error);
    if (error) *error = err;
    return false;
}

bool readImagesGray(const std::vector<std::string>& paths, std::vector<Image8u>& images, std::vector<std::string>* errors, int cuda_device)
{
    const size_t n = paths.size();
    images.assign(n, Image8u());
    std::vector<std::string> errs(n);
    std::vector<std::string> by_kind[3];
    std::vector<size_t> idx[3];
    for (size_t i = 0; i < n; ++i) {
        const int k = image_kind(paths[i], errs[i]);
        by_kind[k].push_back(paths[i]);
        idx[k].push_back(i);
    }
    for (int k = 1; k <= 2; ++k) {
        if (by_kind[k].empty()) continue;
        std::vector<Image8u> im;
        std::vector<std::string> e;
        if (k == 1) readJPEGsGray(by_kind[k], im, &e, cuda_device);
        else readPNGsGray(by_kind[k], im, &e, cuda_device);
        for (size_t j = 0; j < idx[k].size(); ++j) { images[idx[k][j]] = im[j]; errs[idx[k][j]] = e[j]; }
    }
    bool ok = true;
    for (size_t i = 0; i < n; ++i) ok = ok && errs[i].empty();
    if (errors) errors->swap(errs);
    return ok;
}

bool readImageGray(const std::string& path, Image8u& image, std::string* error, int cuda_device)
{
    std::vector<Image8u> images;
    std::vector<std::string> errors;
    const bool ok = readImagesGray(std::vector<std::string>(1, path), images, &errors, cuda_device);
    image = images[0];
    if (!ok && error) *error = errors[0];
    return ok;
}

}  // namespace L3DPP

// C wrappers (include/l3dpp_capi.h): a batch of decoded files is a handle (l3d_image_files.h)
extern "C" {
int l3dpp_png_size(const char* path, int* width, int* height, char* err, int errcap)
{
    std::string e;
    if (!L3DPP::readPNGSize(path, *width, *height, &e)) { l3dpp_copy_str(e, err, errcap); return -1; }
    return 0;
}

void* l3dpp_pngs_read(const char* const* paths, int n, int cuda_device)
{
    L3DImageBatch* b = new L3DImageBatch();
    L3DPP::readPNGsGray(std::vector<std::string>(paths, paths + (n > 0 ? n : 0)), b->images, &b->errors, cuda_device);
    return b;
}

void l3dpp_pngs_close(void* h) { delete (L3DImageBatch*)h; }

int l3dpp_pngs_image(void* h, int i, int* width, int* height, unsigned char* out, long long cap, char* err, int errcap)
{
    return l3d_batch_image(h, i, width, height, out, cap, err, errcap);
}

int l3dpp_image_size(const char* path, int* width, int* height, char* err, int errcap)
{
    std::string e;
    if (!L3DPP::readImageSize(path, *width, *height, &e)) { l3dpp_copy_str(e, err, errcap); return -1; }
    return 0;
}

void* l3dpp_images_read(const char* const* paths, int n, int cuda_device)
{
    L3DImageBatch* b = new L3DImageBatch();
    L3DPP::readImagesGray(std::vector<std::string>(paths, paths + (n > 0 ? n : 0)), b->images, &b->errors, cuda_device);
    return b;
}

void l3dpp_images_close(void* h) { delete (L3DImageBatch*)h; }

int l3dpp_images_image(void* h, int i, int* width, int* height, unsigned char* out, long long cap, char* err, int errcap)
{
    return l3d_batch_image(h, i, width, height, out, cap, err, errcap);
}
}
