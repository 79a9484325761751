// l3d_sfm_handle.h — the object behind an l3dpp_sfm_* handle of the C wrappers (line3d_io.cc, line3d_sfm.cc; tests / Python): the cameras
// of any SfM reader, and the lenses readColmap returns when asked for them.  Host only, header only.
#ifndef L3DPP_SFM_HANDLE_H_
#define L3DPP_SFM_HANDLE_H_
#include "../../include/line3d_io.h"

#include <vector>

struct L3DSfMHandle {
    std::vector<L3DPP::SfMCamera> cams;
    std::vector<L3DPP::LensDistortion> lenses;
};

#endif
