// l3d_png.h — what the PNG chunk parser (line3d_png.cc) hands to the GPU decode (l3d_png.cu): the header of one file, its grey
// conversion and the byte ranges of its IDAT payload.  Host only; DESIGN.md §4d.
#ifndef L3D_PNG_H_
#define L3D_PNG_H_
#include <stdint.h>

#include <string>
#include <utility>
#include <vector>

struct L3DPngHeader {
    int width = 0, height = 0;              // IHDR
    int depth = 0, color_type = 0, interlace = 0, channels = 0;
    int orientation = 1;                    // OpenCV's EXIF orientation, 1..8 (1 when absent, broken or out of range)
    int out_width = 0, out_height = 0;      // imread's output size: the image, transposed for orientations 5..8
    uint8_t palette[768] = {};              // PLTE, zero beyond its entries (indices past it read black, as in libpng)
    bool gamma = false;                     // libpng converts to grey through its gamma tables (gAMA / sRGB on a colour image)
    uint8_t to_linear[256] = {}, from_linear[256] = {};   // those tables: libpng's gamma_to_1 and gamma_from_1
    int window_bits = 15;                   // the zlib header's window (CINFO + 8): a longer distance is corrupt data
    int64_t raw_size = 0;                   // filtered scanlines of every pass, filter bytes included: what the zlib stream must inflate to
    int64_t pass_off[7] = {}, pass_rb[7] = {};          // per Adam7 pass (pass 0 only when not interlaced): offset in the raw bytes, bytes per row
    int pass_w[7] = {}, pass_h[7] = {};
    int64_t zlib_size = 0;                  // the IDAT payload in all: the zlib stream
    std::vector<std::pair<int64_t, int64_t> > idat;     // [first, end) byte offsets of every IDAT payload in the file
};

// Parses a file's chunks.  false with err naming the reason for anything outside the subset of DESIGN.md §4d.
bool l3d_png_parse(const uint8_t* data, int64_t size, L3DPngHeader& h, std::string& err);

#endif
