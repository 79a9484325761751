// l3d_image_files.h — what the JPEG and PNG file readers share (line3d_jpeg.cc, line3d_png.cc): reading a file, decoding a batch of
// files on the GPU with one verdict per file, and the batch handle of their C wrappers (include/l3dpp_capi.h).  Host only, header only.
#ifndef L3D_IMAGE_FILES_H_
#define L3D_IMAGE_FILES_H_
#include "../../include/line3d_io.h"
#include "../../include/l3d_capi.h"
#include "l3dpp_wrap.h"

#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

inline bool l3d_read_file(const std::string& path, std::vector<uint8_t>& bytes, std::string& err)
{
    std::ifstream f(path.c_str(), std::ios::binary);
    if (!f) { err = path + ": cannot open file"; return false; }
    bytes.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
    if (f.bad()) { err = path + ": read error"; return false; }
    return true;
}

// Every readable file of `paths` decoded in one call of `decode` (l3d_decode_jpeg_gray_u8 or l3d_decode_png_gray_u8) on device
// cuda_device.  parse(data, size, out_width, out_height, err) checks one file.  A file that cannot be read, parsed or decoded leaves
// its image empty and its own message in errors[i]; a batch that fails on the GPU is decoded again one file at a time, so that every
// file gets its own verdict.  Returns whether every file was decoded.
template <class Desc, class Parse>
bool l3d_read_gray_files(const std::vector<std::string>& paths, std::vector<L3DPP::Image8u>& images, std::vector<std::string>* errors, int cuda_device,
                         Parse parse, int (*decode)(l3d_ctx*, int, const Desc*, int), const char* format)
{
    const size_t n = paths.size();
    images.assign(n, L3DPP::Image8u());
    std::vector<std::string> errs(n);
    std::vector<std::vector<uint8_t> > files(n);
    std::vector<Desc> descs;
    std::vector<size_t> which;
    for (size_t i = 0; i < n; ++i) {
        int w = 0, h = 0;
        std::string err;
        if (!l3d_read_file(paths[i], files[i], err)) { errs[i] = err; continue; }
        if (!parse(files[i].data(), (int64_t)files[i].size(), w, h, err)) { errs[i] = paths[i] + ": " + err; continue; }
        images[i] = L3DPP::Image8u(h, w, 1);
        Desc d;
        d.data = files[i].data(); d.size = (int64_t)files[i].size();
        d.dst = images[i].data.data(); d.dst_pitch = w;
        d.out_width = w; d.out_height = h;
        descs.push_back(d);
        which.push_back(i);
    }
    if (!descs.empty()) {
        l3d_ctx* ctx = nullptr;
        if (l3d_ctx_create(cuda_device, &ctx) != L3D_OK) {
            for (size_t k : which) {
                errs[k] = paths[k] + ": no usable CUDA device (" + format + " files are decoded on the GPU)";
                images[k] = L3DPP::Image8u();
            }
        } else if (decode(ctx, (int)descs.size(), descs.data(), 0) != L3D_OK) {
            for (size_t j = 0; j < descs.size(); ++j)
                if (decode(ctx, 1, &descs[j], 0) != L3D_OK) {
                    std::string e = l3d_last_error(ctx);
                    const size_t colon = e.find("image 0: ");
                    errs[which[j]] = paths[which[j]] + ": " + (colon == std::string::npos ? e : e.substr(colon + 9));
                    images[which[j]] = L3DPP::Image8u();
                }
        }
        l3d_ctx_destroy(ctx);
    }
    bool ok = true;
    for (size_t i = 0; i < n; ++i) ok = ok && errs[i].empty();
    if (errors) errors->swap(errs);
    return ok;
}

// the handle of l3dpp_jpegs_read, l3dpp_pngs_read and l3dpp_images_read: a batch of decoded files
struct L3DImageBatch {
    std::vector<L3DPP::Image8u> images;
    std::vector<std::string> errors;
};

// file i of a batch: its size, and its packed grey pixels into out[cap] when cap >= width * height; -1 with the file's error in err
inline int l3d_batch_image(void* h, int i, int* width, int* height, unsigned char* out, long long cap, char* err, int errcap)
{
    const L3DImageBatch* b = (const L3DImageBatch*)h;
    if (i < 0 || i >= (int)b->images.size()) { l3dpp_copy_str("no such image", err, errcap); return -1; }
    if (!b->errors[i].empty()) { l3dpp_copy_str(b->errors[i], err, errcap); return -1; }
    const L3DPP::Image8u& im = b->images[i];
    *width = im.cols; *height = im.rows;
    if (out && cap >= (long long)im.data.size()) memcpy(out, im.data.data(), im.data.size());
    return 0;
}

#endif
