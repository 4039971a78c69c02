// What loop_verify.cpp needs of pose_graph.cpp's handles: the batch that owns a graph, its capacity and device, the
// error strings, and the loop-verification state a batch owns (released with the batch).
#pragma once
#include <string>
#include <vector>

#include "vinsb200/pose_graph.h"

namespace vb {
struct LvState;
void lv_release(LvState* s);
LvState** pg_loop_state(vp_batch* b);
vp_batch* pg_owner(vp_graph* g, int* member, bool* standalone);
int pg_capacity(const vp_batch* b, int* device);
std::string* pg_error(vp_graph* g);
std::string* pg_batch_error(vp_batch* b);

// What pose_graph.cpp's vp_save / vp_load need of loop_verify.cpp: the corners, normalised corners and descriptors of a
// member's slots 0 .. kfs.size() - 1 (a slot never attached gives none), and the way back for loaded key frames.
struct MapKeyFrame;
int lv_max_corners(const LvState* s);
int lv_read_points(LvState* s, int member, std::vector<MapKeyFrame>* kfs, std::string* err);
// Writes kfs[i]'s points into slot first + i (n_win = 0, the header pose = P / Q wxyz of key frame i, 3 / 4 per key
// frame) through one staging copy and one scatter launch, then marks the slots attached.
int lv_write_points(LvState* s, int member, int first, const std::vector<MapKeyFrame>& kfs, const double* P, const double* Q,
                    std::string* err);
}  // namespace vb
