// What loop_verify.cpp needs of pose_graph.cpp's handles: the batch that owns a graph, its capacity and device, the
// error strings, and the loop-verification state a batch owns (released with the batch).
#pragma once
#include <string>

#include "vinsb200/pose_graph.h"

namespace vb {
struct LvState;
void lv_release(LvState* s);
LvState** pg_loop_state(vp_batch* b);
vp_batch* pg_owner(vp_graph* g, int* member, bool* standalone);
int pg_capacity(const vp_batch* b, int* device);
std::string* pg_error(vp_graph* g);
std::string* pg_batch_error(vp_batch* b);
}  // namespace vb
