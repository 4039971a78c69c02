// The pose graph's handles, shared by pose_graph.cpp (key frames, optimisation) and loop_verify.cpp (the
// loop-verification state a batch owns, released with the batch), and what vp_save / vp_load need of loop_verify.cpp.
#pragma once
#include <chrono>
#include <string>
#include <vector>

#include "batch_host.h"
#include "cuda_check.h"
#include "rotation.h"
#include "vinsb200/pose_graph.h"

namespace vb {
struct LvState;
void lv_release(LvState* s);

// The corners, normalised corners and descriptors of a member's slots 0 .. kfs.size() - 1 (a slot never attached gives
// none), and the way back for loaded key frames.
struct MapKeyFrame;
int lv_max_corners(const LvState* s);
int lv_read_points(LvState* s, int member, std::vector<MapKeyFrame>* kfs, std::string* err);
// Writes kfs[i]'s points into slot first + i (n_win = 0, the header pose = P / Q wxyz of key frame i, 3 / 4 per key
// frame) through one staging copy and one scatter launch, then marks the slots attached.
int lv_write_points(LvState* s, int member, int first, const std::vector<MapKeyFrame>& kfs, const double* P, const double* Q,
                    std::string* err);

struct PgKeyFrame {
    double stamp = 0;
    Vec3 vio_P, P;
    Mat3 vio_R, R;
    int seq = 0;
    bool has_loop = false;
    int loop_index = -1;
    double loop_info[8] = {};
};
}  // namespace vb

struct vp_graph : vb::MemberBase<vp_batch> {
    vp_config cfg{};
    std::vector<vb::PgKeyFrame> kfs;
    int sequence = 1;      // the node's sequence counter (pose_graph_node.cpp:69-72)
    int sequence_cnt = 0;  // PoseGraph::sequence_cnt
    std::vector<int> sequence_loop{0};
    vb::Mat3 w_r_vio, r_drift;
    vb::Vec3 w_t_vio, t_drift;
    double yaw_drift = 0;
    int earliest_loop_index = -1, pending = -1, n_loops = 0, n_opt = 0;
    int n_map = 0;  // key frames 0 .. n_map - 1 came from vp_load: sequence 0, constant in every optimisation
    // the optimisation in flight (enqueued, not collected): its range, the key frames it packed (global index by local
    // index), the pitch / roll it used, its output once copied
    bool inflight = false, ready = false;
    int inf_first = 0, inf_cur = 0, inf_D = 0;
    std::vector<int> inf_map;
    std::vector<double> inf_pr, inf_out;
    int last_info[4] = {0, 0, 0, 0};
    double last_cost[2] = {0, 0};
    float last_ms = 0;
    int last_launches = 0;
};

struct vp_batch : vb::BatchBase<vp_graph> {
    vp_config cfg{};
    int cap_anchors = 0;  // free loop anchors an optimised range may hold (vp_config::max_anchors, 0 = PG_MAX_ANCHORS)
    vb::PinnedArray<char> h_in;
    vb::DeviceArray<char> d_in;
    vb::PinnedArray<double> h_out;
    vb::DeviceArray<double> d_out, d_work;
    size_t work_stride = 0, in_bytes = 0, out_doubles = 0;
    vb::Stream stream;
    vb::Event ev0, ev1;
    bool busy = false;
    std::vector<int> slots;            // members of the launch in flight, by slot
    std::vector<long long> slot_out;   // their output offsets (doubles)
    std::chrono::steady_clock::time_point t0;
    float ms[2] = {0, 0};
    int launches = 0;
    vb::LvState* lv = nullptr;  // loop verification (loop_verify.cpp), once enabled
};
