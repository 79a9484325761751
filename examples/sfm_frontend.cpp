// examples/sfm_frontend.cpp — the reference's mavmap, OpenMVG, Pix4D and COLMAP frontends (main_mavmap.cpp, main_openmvg.cpp, main_pix4d.cpp,
// main_colmap.cpp) on
// top of include/line3d.h + include/line3d_io.h: read the model, hand every camera its 2D segments, match, reconstruct, save.  Like
// examples/vsfm_frontend.cpp it is deliberately small: no option parser, and the 2D segments come from text files because line
// detection is outside this library.  The images are not loaded either, so lens distortion is only reported: the segments are expected
// in the undistorted image (Line3D::undistortImage with the camera's coefficients, or with its LensDistortion, gives that image).
//
//   sfm_frontend mavmap  <result.txt>     <segments_dir> <output_dir> [const_reg_depth]
//   sfm_frontend openmvg <sfm_data.json>  <segments_dir> <output_dir>
//   sfm_frontend pix4d   <params_folder>  <segments_dir> <output_dir> <project_prefix>
//   sfm_frontend colmap  <sparse folder>  <segments_dir> <output_dir>      (text or binary model; prints every camera's lens)
//   <segments_dir>/<image file name>.txt :  first line "width height", then one "x1 y1 x2 y2" per line
//
// build:  g++ -std=c++17 examples/sfm_frontend.cpp -Iinclude -Lline3dpp_b200 -ll3d_b200 -Wl,-rpath,$PWD/line3dpp_b200 -o sfm_frontend
#include "line3d.h"
#include "line3d_io.h"

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <stdexcept>

static bool read_segments(const std::string& path, int& w, int& h, std::vector<L3DPP::Vec4f>& segs)
{
    std::ifstream f(path.c_str());
    if (!f || !(f >> w >> h)) return false;
    L3DPP::Vec4f s;
    while (f >> s.v[0] >> s.v[1] >> s.v[2] >> s.v[3]) segs.push_back(s);
    return !segs.empty();
}

int main(int argc, char** argv)
{
    const std::string fmt = argc > 1 ? argv[1] : "";
    if (argc < 5 || (fmt != "mavmap" && fmt != "openmvg" && fmt != "pix4d" && fmt != "colmap") || (fmt == "pix4d" && argc < 6)) {
        std::fprintf(stderr, "usage: %s mavmap|openmvg|pix4d|colmap <model> <segments_dir> <output_dir> [const_reg_depth | project_prefix]\n", argv[0]);
        return 2;
    }
    const std::string model = argv[2], segdir = argv[3], outdir = argv[4];
    const bool mavmap = fmt == "mavmap";
    const float const_reg_depth = mavmap && argc > 5 ? (float)std::atof(argv[5]) : -1.0f;

    std::vector<L3DPP::SfMCamera> cams;
    std::vector<L3DPP::LensDistortion> lenses;
    std::string err;
    bool ok;
    if (mavmap) ok = L3DPP::readMavmap(model, cams, &err);
    else if (fmt == "openmvg") ok = L3DPP::readOpenMVG(model, cams, &err);
    else if (fmt == "colmap") ok = L3DPP::readColmap(model, cams, &err, &lenses);   // cameras/images/points3D .txt, or else .bin
    else ok = L3DPP::readPix4D(model, argv[5], cams, &err);             // triangulates the tie points on GPU 0
    if (!ok) { std::fprintf(stderr, "%s\n", err.c_str()); return 1; }
    for (size_t i = 0; i < lenses.size(); ++i) {
        const L3DPP::LensDistortion& l = lenses[i];
        const bool fe = l.model == L3DPP::LensDistortion::FISHEYE;
        std::printf("camera %u (%s): %s lens, k = %g %g %g %g %g %g, p = %g %g\n", cams[i].id, cams[i].image.c_str(), fe ? "fisheye" : "radtan", l.k[0],
                    l.k[1], l.k[2], l.k[3], l.k[4], l.k[5], l.p[0], l.p[1]);
    }

    try {
        // mavmap has no world points: explicit neighbour lists and a constant regularisation depth (main_mavmap.cpp:150-151, 309-326)
        L3DPP::Line3D line3D(outdir, L3DPP::L3D_DEF_LOAD_AND_STORE_SEGMENTS, L3DPP::L3D_DEF_MAX_IMG_WIDTH, L3DPP::L3D_DEF_MAX_NUM_SEGMENTS, !mavmap, true);
        for (size_t i = 0; i < cams.size(); ++i) {
            const L3DPP::SfMCamera& c = cams[i];
            std::string name = c.image;
            const size_t slash = name.find_last_of("/\\");
            if (slash != std::string::npos) name = name.substr(slash + 1);
            int w = 0, h = 0;
            std::vector<L3DPP::Vec4f> segs;
            if (!read_segments(segdir + "/" + name + ".txt", w, h, segs)) { std::fprintf(stderr, "no segments for %s, skipped\n", name.c_str()); continue; }
            bool distorted = c.radial[0] != 0.0 || c.radial[1] != 0.0 || c.radial[2] != 0.0 || c.tangential[0] != 0.0 || c.tangential[1] != 0.0;
            for (int k = 0; k < 6 && i < lenses.size(); ++k) distorted = distorted || lenses[i].k[k] != 0.0;
            if (distorted)
                std::fprintf(stderr, "note: %s is distorted; segments are expected in the undistorted image\n", name.c_str());
            const std::list<unsigned int> list = mavmap ? L3DPP::sequentialNeighbors((unsigned int)i, (unsigned int)cams.size(), L3DPP::L3D_DEF_MATCHING_NEIGHBORS)
                                                        : c.worldpoints;
            if (!line3D.addImage(c.id, w, h, c.K, c.R, c.t, mavmap ? const_reg_depth : c.median_depth, list, segs))
                std::fprintf(stderr, "addImage(%u): %s\n", c.id, line3D.lastError());
        }
        if (line3D.numImages() < 3) { std::fprintf(stderr, "fewer than three usable images\n"); return 1; }
        line3D.matchImages(L3DPP::L3D_DEF_SCORING_POS_REGULARIZER, L3DPP::L3D_DEF_SCORING_ANG_REGULARIZER, L3DPP::L3D_DEF_MATCHING_NEIGHBORS,
                           L3DPP::L3D_DEF_EPIPOLAR_OVERLAP, L3DPP::L3D_DEF_KNN, const_reg_depth);
        if (line3D.lastError()[0]) { std::fprintf(stderr, "matchImages: %s\n", line3D.lastError()); return 1; }
        line3D.reconstruct3Dlines();
        if (line3D.lastError()[0]) { std::fprintf(stderr, "reconstruct3Dlines: %s\n", line3D.lastError()); return 1; }
        std::vector<L3DPP::FinalLine3D> result;
        line3D.get3Dlines(result);
        line3D.saveResultAsSTL(outdir);
        line3D.saveResultAsOBJ(outdir);
        line3D.save3DLinesAsTXT(outdir);
        line3D.save3DLinesAsBIN(outdir);
        std::printf("%zu images, %zu 3D lines -> %s/%s.{stl,obj,txt,bin}\n", line3D.numImages(), result.size(), outdir.c_str(),
                    line3D.createOutputFilename().c_str());
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Line3D++: %s\n", e.what());
        return 3;
    }
    return 0;
}
