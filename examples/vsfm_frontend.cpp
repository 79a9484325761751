// examples/vsfm_frontend.cpp — a VisualSfM frontend on top of include/line3d.h + include/line3d_io.h, in the reference's host
// language, showing what remains of main_vsfm.cpp (reference, 334 lines) when this library is dropped in: read the .nvm model,
// hand every camera its 2D segments, match, reconstruct, save.  Not part of the measured path and deliberately small: no option
// parser, and the 2D segments come from text files because line detection (OpenCV LSD in the reference, line3D.cc:249-372) is
// outside this library.
//
//   vsfm_frontend <model.nvm> <segments_dir> <output_dir> [diffusion 0|1] [collinearity_t px] [bundle 0|1] [devices, e.g. 0,1,2,3]
//   <segments_dir>/<image file name>.txt :  first line "width height", then one "x1 y1 x2 y2" per line
//   devices: CUDA devices to match on (default 0); the first one also runs everything after matching
//
// build:  g++ -std=c++17 examples/vsfm_frontend.cpp -Iinclude -Lline3dpp_b200 -ll3d_b200 -Wl,-rpath,$PWD/line3dpp_b200 -o vsfm_frontend
#include "line3d.h"
#include "line3d_io.h"

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>
#include <stdexcept>

static bool read_segments(const std::string& path, int& w, int& h, std::vector<L3DPP::Vec4f>& segs)
{
    std::ifstream f(path.c_str());
    if (!f || !(f >> w >> h)) return false;
    L3DPP::Vec4f s;
    while (f >> s.v[0] >> s.v[1] >> s.v[2] >> s.v[3]) segs.push_back(s);
    return !segs.empty();
}

// "0,1,2" -> {0, 1, 2}; false for anything else
static bool parse_devices(const std::string& list, std::vector<int>& out)
{
    std::stringstream s(list);
    std::string item;
    while (std::getline(s, item, ',')) {
        char* end = nullptr;
        const long d = std::strtol(item.c_str(), &end, 10);
        if (item.empty() || *end || d < 0) return false;
        out.push_back((int)d);
    }
    return !out.empty();
}

int main(int argc, char** argv)
{
    if (argc < 4) { std::fprintf(stderr, "usage: %s <model.nvm> <segments_dir> <output_dir> [diffusion 0|1] [collinearity_t] [bundle 0|1] [devices]\n", argv[0]); return 2; }
    const std::string nvm = argv[1], segdir = argv[2], outdir = argv[3];
    const bool diffusion = argc > 4 && std::atoi(argv[4]) != 0;
    const float collinearity = argc > 5 ? (float)std::atof(argv[5]) : L3DPP::L3D_DEF_COLLINEARITY_T;
    const bool bundle = argc > 6 && std::atoi(argv[6]) != 0;
    std::vector<int> devices;
    if (argc <= 7) devices.push_back(0);
    else if (!parse_devices(argv[7], devices)) { std::fprintf(stderr, "bad device list '%s'\n", argv[7]); return 2; }

    std::vector<L3DPP::NVMCamera> cams;
    std::string err;
    if (!L3DPP::readNVM(nvm, cams, &err)) { std::fprintf(stderr, "%s\n", err.c_str()); return 1; }     // main_vsfm.cpp:143-250

    try {
        // main_vsfm.cpp:128-141: neighbours by world points, GPU on (there is no CPU fallback in this library), on every listed device
        L3DPP::Line3D line3D(outdir, L3DPP::L3D_DEF_LOAD_AND_STORE_SEGMENTS, L3DPP::L3D_DEF_MAX_IMG_WIDTH, L3DPP::L3D_DEF_MAX_NUM_SEGMENTS, true, true, devices);
        for (size_t i = 0; i < cams.size(); ++i) {                                                     // main_vsfm.cpp:252-310
            const L3DPP::NVMCamera& c = cams[i];
            if (c.worldpoints.empty()) continue;
            std::string name = c.image;
            const size_t slash = name.find_last_of("/\\");
            if (slash != std::string::npos) name = name.substr(slash + 1);
            int w = 0, h = 0;
            std::vector<L3DPP::Vec4f> segs;
            if (!read_segments(segdir + "/" + name + ".txt", w, h, segs)) { std::fprintf(stderr, "no segments for %s, skipped\n", name.c_str()); continue; }
            if (c.distortion != 0.0f) std::fprintf(stderr, "note: %s has radial distortion %g; segments are expected in the undistorted image\n", name.c_str(), c.distortion);
            if (!line3D.addImage((unsigned int)i, w, h, L3DPP::intrinsicsFromFocal(c.focal, w, h), c.R, c.t, c.median_depth, c.worldpoints, segs))
                std::fprintf(stderr, "addImage(%zu): %s\n", i, line3D.lastError());
        }
        if (line3D.numImages() < 3) { std::fprintf(stderr, "fewer than three usable images\n"); return 1; }
        line3D.matchImages();                                                                           // main_vsfm.cpp:313-315, defaults
        if (line3D.lastError()[0]) { std::fprintf(stderr, "matchImages: %s\n", line3D.lastError()); return 1; }
        line3D.reconstruct3Dlines(L3DPP::L3D_DEF_MIN_VISIBILITY_T, diffusion, collinearity, bundle);      // main_vsfm.cpp:318-319
        if (line3D.lastError()[0]) { std::fprintf(stderr, "reconstruct3Dlines: %s\n", line3D.lastError()); return 1; }
        std::vector<L3DPP::FinalLine3D> result;
        line3D.get3Dlines(result);
        line3D.saveResultAsSTL(outdir);                                                                 // main_vsfm.cpp:325-330
        line3D.saveResultAsOBJ(outdir);
        line3D.save3DLinesAsTXT(outdir);
        const L3DPP::Line3DStats& st = line3D.stats();
        std::printf("%zu images, %lld view pairs, %lld pair evaluations, %zu 3D lines -> %s/%s.{stl,obj,txt}\n", line3D.numImages(), st.view_pairs,
                    st.pair_evaluations, result.size(), outdir.c_str(), line3D.createOutputFilename().c_str());
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Line3D++: %s\n", e.what());
        return 3;
    }
    return 0;
}
