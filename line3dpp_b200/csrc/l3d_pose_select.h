// l3d_pose_select.h — the host half of l3d_pose_neighbors (csrc/l3d_pose.cu): the selection of find_visual_neighbors
// (csrc/line3d_host.cc) over candidates the device has ranked
#pragma once
#include "../../include/l3d_capi.h"

#include <vector>

namespace L3DPP {

struct PoseCandidate { unsigned int cam; float score; };

// view i's candidates (common > 4) are cand[cand_off[i] .. cand_off[i+1]), by score descending, ties in ascending camID; out[i] gets
// its neighbours' camIDs in ascending order.  Camera centres, axes and distances come from each view's K, R, t as addImage computes them.
void pose_select_neighbors(int n, const l3d_pose_view* views, const long long* cand_off, const PoseCandidate* cand, unsigned int num_neighbors,
                           std::vector<std::vector<unsigned int> >& out);

}  // namespace L3DPP
