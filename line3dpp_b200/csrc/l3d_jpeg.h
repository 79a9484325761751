// l3d_jpeg.h — what the JPEG marker parser (line3d_jpeg.cc) hands to the GPU decode (l3d_jpeg.cu): the header of one file and the
// byte ranges of the entropy-coded segments of the scan that carries Y.  Host only; DESIGN.md §4c.
#ifndef L3D_JPEG_H_
#define L3D_JPEG_H_
#include <stdint.h>

#include <string>
#include <utility>
#include <vector>

// one DHT table as the file gives it: bits[l-1] codes of length l, then the symbols in code order
struct L3DJpegHuffSpec {
    uint8_t bits[16];
    uint8_t vals[256];
};

struct L3DJpegHeader {
    int width = 0, height = 0;             // the frame as coded
    int orientation = 1;                    // OpenCV's EXIF orientation, 1..8 (1 when absent, broken or out of range)
    int out_width = 0, out_height = 0;      // imread's output size: the frame, transposed for orientations 5..8
    // the scan that carries Y (component 0 of the frame)
    int ns = 0, y_in_scan = 0;              // components in the scan, Y's position among them
    int mcus_x = 0, mcus = 0;               // MCUs per row and in all; one block per MCU in a non-interleaved scan
    int restart = 0;                        // MCUs per entropy-coded segment (the DRI interval; 0: one segment)
    int bh[4] = {1, 1, 1, 1}, bv[4] = {1, 1, 1, 1};    // blocks of scan component k per MCU: its sampling factors when interleaved
    L3DJpegHuffSpec dc[4], ac[4];           // the tables of scan component k when the scan starts
    uint16_t q[64];                         // Y's quantisation table (natural order) when its scan starts
    int yblocks_x = 0, yblocks_y = 0;       // Y's coded block grid (MCU-padded when interleaved)
    std::vector<std::pair<int64_t, int64_t> > segs;    // [first, end) byte offsets of every segment; fill bytes and markers excluded
};

// Parses a file's markers.  false with err naming the reason for anything outside the subset of DESIGN.md §4c.
bool l3d_jpeg_parse(const uint8_t* data, int64_t size, L3DJpegHeader& h, std::string& err);

#endif
