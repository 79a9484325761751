// l3d_exif.h — OpenCV's EXIF orientation, shared by the JPEG and PNG readers (DESIGN.md §4c, §4d): the orientation tag of a TIFF
// block, and the orientation as an affine map of pixel positions.  Host only.
#ifndef L3D_EXIF_H_
#define L3D_EXIF_H_
#include <stdint.h>

#include <cstring>

// OpenCV's ExifReader on a TIFF block (a JPEG APP1 payload after "Exif\0\0", a PNG eXIf chunk): IFD0's tag 0x0112 as a 16-bit value
// in the TIFF byte order; 0 when the block is broken or has no such tag (both mean: no transform)
inline int l3d_exif_orientation(const uint8_t* p, int64_t n)
{
    if (n < 8 || !((p[0] == 'I' && p[1] == 'I') || (p[0] == 'M' && p[1] == 'M'))) return 0;
    const bool be = p[0] == 'M';
    auto u16 = [&](int64_t o) { return be ? (p[o] << 8 | p[o + 1]) : (p[o + 1] << 8 | p[o]); };
    auto u32 = [&](int64_t o) { return be ? ((uint32_t)u16(o) << 16 | (uint32_t)u16(o + 2)) : ((uint32_t)u16(o + 2) << 16 | (uint32_t)u16(o)); };
    if (u16(2) != 0x2A) return 0;
    const int64_t off = u32(4);
    if (off + 2 > n) return 0;
    const int count = u16(off);
    for (int i = 0; i < count; ++i) {
        const int64_t e = off + 2 + 12 * (int64_t)i;
        if (e + 12 > n) return 0;
        if (u16(e) == 0x0112) return u16(e + 8);
    }
    return 0;
}

// orientation o (1..8) as an affine map of (y, x) in a W x H frame (OpenCV's ExifTransform): the pixel goes to row
// a[0]*y + a[1]*x + a[2], column a[3]*y + a[4]*x + a[5]
inline void l3d_orientation_map(int o, int W, int H, int a[6])
{
    int b[6] = {1, 0, 0, 0, 1, 0};
    switch (o) {
    case 2: { int t[6] = {1, 0, 0, 0, -1, W - 1}; memcpy(b, t, sizeof(b)); break; }
    case 3: { int t[6] = {-1, 0, H - 1, 0, -1, W - 1}; memcpy(b, t, sizeof(b)); break; }
    case 4: { int t[6] = {-1, 0, H - 1, 0, 1, 0}; memcpy(b, t, sizeof(b)); break; }
    case 5: { int t[6] = {0, 1, 0, 1, 0, 0}; memcpy(b, t, sizeof(b)); break; }
    case 6: { int t[6] = {0, 1, 0, -1, 0, H - 1}; memcpy(b, t, sizeof(b)); break; }
    case 7: { int t[6] = {0, -1, W - 1, -1, 0, H - 1}; memcpy(b, t, sizeof(b)); break; }
    case 8: { int t[6] = {0, -1, W - 1, 1, 0, 0}; memcpy(b, t, sizeof(b)); break; }
    default: break;
    }
    memcpy(a, b, sizeof(b));
}

#endif
