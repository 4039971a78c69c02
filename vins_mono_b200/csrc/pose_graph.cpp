// Host bookkeeping of the pose graph (include/vinsb200/pose_graph.h): PoseGraph::addKeyFrame, updateKeyFrameLoop and the
// before / after parts of optimize4DoF (pose_graph/src/pose_graph.cpp) around the device solve of pg_kernels.cu.
#include "vinsb200/pose_graph.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "cuda_check.h"
#include "host_math.h"
#include "pg_host.h"
#include "pg_kernels.h"
#include "pg_layout.h"
#include "pg_map.h"

using hm::Mat3;
using hm::Quat;
using hm::Vec3;

namespace {

constexpr int PG_MAX_ITERATIONS = 5;  // options.max_num_iterations, pose_graph.cpp:437

struct KeyFrame {
    double stamp = 0;
    Vec3 vio_P, P;
    Mat3 vio_R, R;
    int seq = 0;
    bool has_loop = false;
    int loop_index = -1;
    double loop_info[8] = {};
};

bool loop_gate(const double* li) {  // keyframe.cpp:480, :573
    return std::fabs(li[7]) < 30.0 && Vec3(li[0], li[1], li[2]).norm() < 20.0;
}

Mat3 yaw_R(double yaw) { return hm::ypr2R(Vec3(yaw, 0, 0)); }

}  // namespace

struct vp_graph {
    vp_batch* owner = nullptr;
    int member = 0;
    bool standalone = false;
    vp_config cfg{};
    std::string err;
    std::vector<KeyFrame> kfs;
    int sequence = 1;      // the node's sequence counter (pose_graph_node.cpp:69-72)
    int sequence_cnt = 0;  // PoseGraph::sequence_cnt
    std::vector<int> sequence_loop{0};
    Mat3 w_r_vio, r_drift;
    Vec3 w_t_vio, t_drift;
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

struct vp_batch {
    vp_config cfg{};
    int S = 0;
    int cap_anchors = 0;  // free loop anchors an optimised range may hold (vp_config::max_anchors, 0 = PG_MAX_ANCHORS)
    std::string err;
    std::vector<vp_graph*> members;
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

namespace {

// Waits for the batch's launch in flight and copies each member's output block to the member (not yet applied).
int batch_wait(vp_batch* b) {
    if (!b->busy) return 0;
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaStreamSynchronize(b->stream));
    b->busy = false;
    float ms = 0;
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaEventElapsedTime(&ms, b->ev0, b->ev1));
    b->ms[0] = ms;
    b->ms[1] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - b->t0).count();
    for (size_t s = 0; s < b->slots.size(); s++) {
        vp_graph* g = b->members[b->slots[s]];
        const int n = (int)g->inf_map.size();
        const double* o = b->h_out + b->slot_out[s];
        g->inf_out.assign(o, o + vb::pg_out_layout(n).total);
        g->ready = true;
        g->last_ms = ms;
        g->last_launches = b->launches;
    }
    b->slots.clear();
    return 0;
}

// Applies the member's collected result: optimize4DoF after ceres::Solve (pose_graph.cpp:532-573).
int collect(vp_graph* g) {
    if (!g->inflight) return 0;
    if (!g->ready) {
        const int rc = batch_wait(g->owner);
        if (rc) {
            g->err = g->owner->err;
            return rc;
        }
    }
    const int first = g->inf_first, cur = g->inf_cur, n = (int)g->inf_map.size();
    if (!g->ready || g->inf_out.size() != vb::pg_out_layout(n).total) {
        g->err = "vp: the optimisation in flight has no result";
        return VP_ERR_CUDA;
    }
    const double* o = g->inf_out.data();
    for (int i = 0; i < n; i++) {
        KeyFrame& kf = g->kfs[g->inf_map[i]];
        if (kf.seq == 0) continue;
        kf.R = hm::ypr2R(Vec3(o[4 * i], g->inf_pr[2 * i], g->inf_pr[2 * i + 1]));
        kf.P = Vec3(o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
    }
    // the loaded map's key frames of the range, packed or not: updatePose(t, ypr2R(euler)) of a constant block
    for (int k = first; k < g->n_map; k++) {
        KeyFrame& kf = g->kfs[k];
        kf.R = hm::ypr2R(hm::R2ypr(Quat::FromR(kf.vio_R).R()));
        kf.P = kf.vio_P;
    }
    const KeyFrame& ck = g->kfs[cur];
    g->yaw_drift = hm::R2ypr(ck.R).x - hm::R2ypr(ck.vio_R).x;
    g->r_drift = yaw_R(g->yaw_drift);
    g->t_drift = ck.P - g->r_drift * ck.vio_P;
    for (size_t k = cur + 1; k < g->kfs.size(); k++) {
        KeyFrame& kf = g->kfs[k];
        kf.P = g->r_drift * kf.vio_P + g->t_drift;
        kf.R = g->r_drift * kf.vio_R;
    }
    const double* sm = o + vb::pg_out_layout(n).summary;
    g->last_info[0] = cur - first + 1;
    g->last_info[1] = g->inf_D;
    g->last_info[2] = (int)sm[0];
    g->last_info[3] = (int)sm[1];
    g->last_cost[0] = sm[2];
    g->last_cost[1] = sm[3];
    g->n_opt++;
    g->inflight = g->ready = false;
    return 0;
}

void release(vp_batch* b) {
    cudaSetDevice(b->cfg.device);
    vb::lv_release(b->lv);
    if (b->stream) cudaStreamSynchronize(b->stream);
    for (vp_graph* g : b->members) delete g;
    delete b;
}

int batch_create(const vp_config* cfg, int n, vp_batch** out) {
    *out = nullptr;
    if (!cfg || n < 1 || cfg->max_keyframes < 2 || cfg->max_anchors < 0 || cfg->max_anchors > vb::PG_CAP_ANCHORS) return VP_ERR_INVALID;
    if (!vb::device_available(cfg->device)) return VP_ERR_NO_DEVICE;
    std::unique_ptr<vp_batch, void (*)(vp_batch*)> b(new vp_batch, release);
    b->cfg = *cfg;
    b->S = n;
    b->cap_anchors = cfg->max_anchors ? cfg->max_anchors : vb::PG_MAX_ANCHORS;
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaSetDevice(cfg->device));
    const int cap = cfg->max_keyframes;
    b->work_stride = (vb::pg_work_layout(cap, b->cap_anchors).total + 1) & ~(size_t)1;
    b->in_bytes = vb::pg_arena_bytes(n, cap, b->cap_anchors);
    b->out_doubles = (size_t)n * vb::pg_out_layout(cap).total;
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->stream.create());
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->ev0.create());
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->ev1.create());
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->h_in.alloc(b->in_bytes));
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->h_out.alloc(b->out_doubles));
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->d_in.alloc(b->in_bytes));
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->d_out.alloc(b->out_doubles));
    VB_CUDA_CHECK(b, VP_ERR_CUDA, b->d_work.alloc((size_t)n * b->work_stride));
    for (int k = 0; k < n; k++) {
        vp_graph* g = new vp_graph;
        g->owner = b.get();
        g->member = k;
        g->cfg = *cfg;
        b->members.push_back(g);
    }
    *out = b.release();
    return 0;
}

// Packs member g's pending optimisation into the input arena at byte offset `off`.  Fails (changing nothing) when its
// range has more free loop anchors than the graph's anchor capacity.
// The range [first, cur] is packed as the solve's local key frames 0 .. n - 1, the nc constant ones first:
//   - without a loaded map in the range (first >= n_map), the range itself; local 0 (first) is the one constant.
//   - with one (first < n_map), the map key frames first .. n_map - 1 are constant, and so are the edges between two of
//     them (sequential edges inside the map, loops stored with it): Ceres drops those from the minimiser.  Only the map
//     key frames that a free key frame's loop lands on are packed, in ascending order and each with a sequence of its
//     own (-1 - j), so that no sequential edge pairs two of them; the free key frames n_map .. cur follow.  The chain's
//     serial work then grows with the free key frames only.
// map (out) receives the global index of each local key frame, pr the pitch and roll of each (the constants of the
// solve).  The member itself is not changed.
int pack_member(vp_graph* g, char* base, size_t off, int* n_out, int* nb_out, int* nc_out, std::vector<int>* map, std::vector<double>* pr) {
    const int first = g->earliest_loop_index, cur = g->pending;
    std::vector<int>& gl = *map;
    gl.clear();
    int nc = 1, seq_base = first;  // local i >= nc holds global seq_base + i - nc
    if (first < g->n_map) {
        for (int k = g->n_map; k <= cur; k++) {
            const KeyFrame& kf = g->kfs[k];
            if (kf.has_loop && kf.loop_index < g->n_map) gl.push_back(kf.loop_index);
        }
        std::sort(gl.begin(), gl.end());
        gl.erase(std::unique(gl.begin(), gl.end()), gl.end());
        nc = (int)gl.size();
        seq_base = g->n_map;
    } else {
        gl.push_back(first);
        seq_base = first + 1;
    }
    for (int k = seq_base; k <= cur; k++) gl.push_back(k);
    const int n = (int)gl.size();
    auto local = [&](int k) {
        return k >= seq_base ? nc + k - seq_base : (int)(std::lower_bound(gl.begin(), gl.begin() + nc, k) - gl.begin());
    };
    std::vector<int> anchors;
    for (int i = nc; i < n; i++) {
        const KeyFrame& kf = g->kfs[gl[i]];
        if (kf.has_loop && local(kf.loop_index) >= nc) anchors.push_back(local(kf.loop_index));
    }
    std::sort(anchors.begin(), anchors.end());
    anchors.erase(std::unique(anchors.begin(), anchors.end()), anchors.end());
    const int nb = (int)anchors.size();
    const int cap = g->owner->cap_anchors;
    if (nb > cap) {
        g->err = "vp_optimize: " + std::to_string(nb) + " free loop anchors in the optimised range, at most " + std::to_string(cap);
        return VP_ERR_CAPACITY;
    }
    const bool map_range = first < g->n_map;
    const vb::PgInLayout il = vb::pg_in_layout(n, nb);
    char* in = base + off;
    double* pose = reinterpret_cast<double*>(in + il.pose);
    double* loopm = reinterpret_cast<double*>(in + il.loop);
    int* seq = reinterpret_cast<int*>(in + il.seq);
    int* loop = reinterpret_cast<int*>(in + il.loop_idx);
    int* bslot = reinterpret_cast<int*>(in + il.bslot);
    int* lfirst = reinterpret_cast<int*>(in + il.lfirst);
    int* lnext = reinterpret_cast<int*>(in + il.lnext);
    int* anc = reinterpret_cast<int*>(in + il.anchors);
    std::vector<int> last(n, -1);
    pr->resize(2 * (size_t)n);
    for (int i = 0; i < n; i++) {
        const KeyFrame& kf = g->kfs[gl[i]];
        const bool packed_edges = !map_range || i >= nc;  // a packed map key frame owns no edge
        const Quat q = Quat::FromR(kf.vio_R);
        const double p[7] = {kf.vio_P.x, kf.vio_P.y, kf.vio_P.z, q.w, q.x, q.y, q.z};
        std::memcpy(pose + 7 * i, p, sizeof(p));
        const Vec3 ypr = hm::R2ypr(q.R());
        (*pr)[2 * i] = ypr.y;
        (*pr)[2 * i + 1] = ypr.z;
        seq[i] = packed_edges ? kf.seq : -1 - i;
        loop[i] = packed_edges && kf.has_loop ? local(kf.loop_index) : -1;
        loopm[4 * i] = kf.loop_info[0];
        loopm[4 * i + 1] = kf.loop_info[1];
        loopm[4 * i + 2] = kf.loop_info[2];
        loopm[4 * i + 3] = kf.loop_info[7];
        bslot[i] = -1;
        lfirst[i] = lnext[i] = -1;
    }
    for (int k = 0; k < nb; k++) {
        anc[k] = anchors[k];
        bslot[anchors[k]] = k;
    }
    for (int i = 0; i < n; i++) {
        const int l = loop[i];
        if (l < 0) continue;
        if (lfirst[l] < 0) lfirst[l] = i;
        else lnext[last[l]] = i;
        last[l] = i;
    }
    *n_out = n;
    *nb_out = nb;
    *nc_out = nc;
    return 0;
}

// One host-to-device copy of the packed arena, the launch chain, one device-to-host copy of the outputs.
int enqueue(vp_batch* b, size_t in_bytes, size_t out_doubles, int count, int max_n, int max_D) {
    b->t0 = std::chrono::steady_clock::now();
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaSetDevice(b->cfg.device));
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaMemcpyAsync(b->d_in, b->h_in, in_bytes, cudaMemcpyHostToDevice, b->stream));
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaEventRecord(b->ev0, b->stream));
    vb::PgLaunch L{b->d_in,           b->d_work, b->work_stride, b->d_out, b->S, b->cfg.max_keyframes,
                   b->cap_anchors, count,     max_n,          max_D,    PG_MAX_ITERATIONS};
    const int launches = vb::launch_pg_optimize(L, b->stream);
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaGetLastError());  // incl. the failed opt-in of a chain that was not launched
    VB_CUDA_CHECK(b, VP_ERR_CUDA, launches < 0 ? cudaErrorInvalidConfiguration : cudaSuccess);
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaEventRecord(b->ev1, b->stream));
    VB_CUDA_CHECK(b, VP_ERR_CUDA, cudaMemcpyAsync(b->h_out, b->d_out, out_doubles * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    b->launches = launches;
    return 0;
}

int batch_optimize(vp_batch* b, const int* active, int* status) {
    int first_err = 0;
    if (batch_wait(b)) return VP_ERR_CUDA;
    const vb::PgHdrLayout hl = vb::pg_hdr_layout(b->S);
    size_t off = hl.total, out_off = 0;
    int count = 0, max_n = 0, max_D = 0;
    int* h_member = reinterpret_cast<int*>(b->h_in + hl.member);
    int* h_n = reinterpret_cast<int*>(b->h_in + hl.n);
    int* h_nb = reinterpret_cast<int*>(b->h_in + hl.nb);
    long long* h_in_off = reinterpret_cast<long long*>(b->h_in + hl.in_off);
    long long* h_out_off = reinterpret_cast<long long*>(b->h_in + hl.out_off);
    int* h_nc = reinterpret_cast<int*>(b->h_in + hl.nc);
    // the members of this launch; their state changes only once the whole chain has been enqueued
    struct Slot {
        int k, nb;
        long long out_off;
        std::vector<int> map;
        std::vector<double> pr;
    };
    std::vector<Slot> slots;
    for (int k = 0; k < b->S; k++) {
        if (status) status[k] = 0;
        vp_graph* g = b->members[k];
        if ((active && !active[k]) || g->pending < 0) continue;
        int rc = collect(g);  // the member's previous result first
        int n = 0, nb = 0, nc = 0;
        std::vector<int> map;
        std::vector<double> pr;
        if (!rc) rc = pack_member(g, b->h_in, off, &n, &nb, &nc, &map, &pr);
        if (rc) {
            if (status) status[k] = rc;
            if (!first_err) first_err = rc;
            continue;
        }
        h_member[count] = k;
        h_n[count] = n;
        h_nb[count] = nb;
        h_nc[count] = nc;
        h_in_off[count] = (long long)off;
        h_out_off[count] = (long long)out_off;
        slots.push_back(Slot{k, nb, (long long)out_off, std::move(map), std::move(pr)});
        off += vb::pg_in_layout(n, nb).total;
        out_off += vb::pg_out_layout(n).total;
        max_n = std::max(max_n, n);
        max_D = std::max(max_D, 4 * nb);
        count++;
    }
    if (!count) return first_err;
    reinterpret_cast<int*>(b->h_in.get())[0] = count;
    const int rc = enqueue(b, off, out_off, count, max_n, max_D);
    if (rc) {  // nothing was committed: every member keeps its pending optimisation
        // the stream may hold part of the chain: it is drained so that a later launch starts clean
        cudaStreamSynchronize(b->stream);
        cudaGetLastError();
        for (const Slot& sl : slots) {
            if (status) status[sl.k] = rc;
            b->members[sl.k]->err = b->err;
        }
        return rc;
    }
    b->slots.clear();
    b->slot_out.clear();
    for (Slot& sl : slots) {
        vp_graph* g = b->members[sl.k];
        b->slots.push_back(sl.k);
        b->slot_out.push_back(sl.out_off);
        g->inflight = true;
        g->ready = false;
        g->inf_first = g->earliest_loop_index;
        g->inf_cur = g->pending;
        g->inf_D = 4 * sl.nb;
        g->inf_map = std::move(sl.map);
        g->inf_pr = std::move(sl.pr);
        g->pending = -1;
        if (status) status[sl.k] = 1;
    }
    b->busy = true;
    return first_err;
}

void store_pose(const KeyFrame& kf, double* P3, double* Q4) {
    if (P3) { P3[0] = kf.P.x; P3[1] = kf.P.y; P3[2] = kf.P.z; }
    if (Q4) {
        const Quat q = Quat::FromR(kf.R);
        Q4[0] = q.w; Q4[1] = q.x; Q4[2] = q.y; Q4[3] = q.z;
    }
}

}  // namespace

namespace vb {
LvState** pg_loop_state(vp_batch* b) { return &b->lv; }
vp_batch* pg_owner(vp_graph* g, int* member, bool* standalone) {
    *member = g->member;
    *standalone = g->standalone;
    return g->owner;
}
int pg_capacity(const vp_batch* b, int* device) {
    *device = b->cfg.device;
    return b->cfg.max_keyframes;
}
std::string* pg_error(vp_graph* g) { return &g->err; }
std::string* pg_batch_error(vp_batch* b) { return &b->err; }
}  // namespace vb

extern "C" {

int vp_create(const vp_config* cfg, vp_graph** out) {
    if (!out) return VP_ERR_INVALID;
    vp_batch* b = nullptr;
    const int rc = batch_create(cfg, 1, &b);
    if (rc) return rc;
    b->members[0]->standalone = true;
    *out = b->members[0];
    return 0;
}

void vp_destroy(vp_graph* g) {
    if (g && g->standalone) release(g->owner);
}

const char* vp_last_error(const vp_graph* g) { return g ? g->err.c_str() : "null handle"; }

int vp_new_sequence(vp_graph* g) {
    if (!g) return VP_ERR_INVALID;
    if (!g->kfs.empty() && g->kfs.back().seq == g->sequence) g->sequence++;
    return 0;
}

int vp_add_keyframe(vp_graph* g, double stamp, const double* vio_P3, const double* vio_Qwxyz, int loop_index, const double* loop_info8,
                    int* index, double* P3, double* Qwxyz) {
    if (!g || !vio_P3 || !vio_Qwxyz || (loop_index >= 0 && !loop_info8)) return VP_ERR_INVALID;
    if ((int)g->kfs.size() >= g->cfg.max_keyframes) {
        g->err = "vp_add_keyframe: the graph holds max_keyframes = " + std::to_string(g->cfg.max_keyframes) + " key frames";
        return VP_ERR_CAPACITY;
    }
    const int idx = (int)g->kfs.size();
    if (loop_index >= idx) {
        g->err = "vp_add_keyframe: loop_index must name an earlier key frame";
        return VP_ERR_INVALID;
    }
    KeyFrame kf;
    kf.stamp = stamp;
    kf.seq = g->sequence;
    if (g->sequence_cnt != kf.seq) {  // pose_graph.cpp:47-57
        g->sequence_cnt++;
        g->sequence_loop.push_back(0);
        g->w_t_vio = Vec3();
        g->w_r_vio = Mat3();
        g->t_drift = Vec3();
        g->r_drift = Mat3();
    }
    const Mat3 R_in = Quat(vio_Qwxyz[0], vio_Qwxyz[1], vio_Qwxyz[2], vio_Qwxyz[3]).R();
    kf.vio_P = g->w_r_vio * Vec3(vio_P3[0], vio_P3[1], vio_P3[2]) + g->w_t_vio;
    kf.vio_R = g->w_r_vio * R_in;
    if (loop_index >= 0 && loop_gate(loop_info8)) {  // findConnection accepted the loop
        kf.has_loop = true;
        kf.loop_index = loop_index;
        std::memcpy(kf.loop_info, loop_info8, sizeof(kf.loop_info));
        if (g->earliest_loop_index > loop_index || g->earliest_loop_index == -1) g->earliest_loop_index = loop_index;
        const KeyFrame& old = g->kfs[loop_index];
        const Vec3 rel_t(loop_info8[0], loop_info8[1], loop_info8[2]);
        const Mat3 rel_R = Quat(loop_info8[3], loop_info8[4], loop_info8[5], loop_info8[6]).R();
        const Vec3 w_P_cur = old.vio_R * rel_t + old.vio_P;
        const Mat3 w_R_cur = old.vio_R * rel_R;
        const double shift_yaw = hm::R2ypr(w_R_cur).x - hm::R2ypr(kf.vio_R).x;
        const Mat3 shift_r = yaw_R(shift_yaw);
        const Vec3 shift_t = w_P_cur - w_R_cur * kf.vio_R.T() * kf.vio_P;
        if (old.seq != kf.seq && g->sequence_loop[kf.seq] == 0) {  // pose_graph.cpp:96-124
            g->w_r_vio = shift_r;
            g->w_t_vio = shift_t;
            kf.vio_P = shift_r * kf.vio_P + shift_t;
            kf.vio_R = shift_r * kf.vio_R;
            for (KeyFrame& o : g->kfs)
                if (o.seq == kf.seq) {
                    o.vio_P = shift_r * o.vio_P + shift_t;
                    o.vio_R = shift_r * o.vio_R;
                }
            g->sequence_loop[kf.seq] = 1;
        }
        g->pending = idx;
        g->n_loops++;
    }
    kf.P = g->r_drift * kf.vio_P + g->t_drift;
    kf.R = g->r_drift * kf.vio_R;
    g->kfs.push_back(kf);
    if (index) *index = idx;
    store_pose(kf, P3, Qwxyz);
    return 0;
}

int vp_update_loop(vp_graph* g, int index, const double* loop_info8) {
    if (!g || !loop_info8 || index < 0 || index >= (int)g->kfs.size() || !g->kfs[index].has_loop) return VP_ERR_INVALID;
    if (!loop_gate(loop_info8)) return 0;
    if (g->cfg.fast_relocalization) {
        const int rc = collect(g);
        if (rc) return rc;
    }
    KeyFrame& kf = g->kfs[index];
    std::memcpy(kf.loop_info, loop_info8, sizeof(kf.loop_info));
    if (g->cfg.fast_relocalization) {  // pose_graph.cpp:895-921
        const KeyFrame& old = g->kfs[kf.loop_index];
        const Vec3 rel_t(loop_info8[0], loop_info8[1], loop_info8[2]);
        const Mat3 rel_R = Quat(loop_info8[3], loop_info8[4], loop_info8[5], loop_info8[6]).R();
        const Vec3 w_P_cur = old.R * rel_t + old.P;
        const Mat3 w_R_cur = old.R * rel_R;
        g->yaw_drift = hm::R2ypr(w_R_cur).x - hm::R2ypr(kf.vio_R).x;
        g->r_drift = yaw_R(g->yaw_drift);
        g->t_drift = w_P_cur - w_R_cur * kf.vio_R.T() * kf.vio_P;
    }
    return 0;
}

int vp_optimize(vp_graph* g) {
    if (!g) return VP_ERR_INVALID;
    std::vector<int> active(g->owner->S, 0), status(g->owner->S, 0);
    active[g->member] = 1;
    const int rc = batch_optimize(g->owner, active.data(), status.data());
    if (rc && g->err.empty()) g->err = g->owner->err;
    return rc ? rc : status[g->member];
}

int vp_sync(vp_graph* g) { return g ? collect(g) : VP_ERR_INVALID; }

int vp_correct_pose(vp_graph* g, const double* P3, const double* Q4, double* P_out3, double* Q_out4) {
    if (!g || !P3 || !Q4) return VP_ERR_INVALID;
    const int rc = collect(g);
    if (rc) return rc;
    KeyFrame t;
    const Vec3 P = g->w_r_vio * Vec3(P3[0], P3[1], P3[2]) + g->w_t_vio;
    const Mat3 R = g->w_r_vio * Quat(Q4[0], Q4[1], Q4[2], Q4[3]).R();
    t.P = g->r_drift * P + g->t_drift;
    t.R = g->r_drift * R;
    store_pose(t, P_out3, Q_out4);
    return 0;
}

int vp_get_drift(vp_graph* g, double* r9, double* t3, double* yaw) {
    if (!g) return VP_ERR_INVALID;
    const int rc = collect(g);
    if (rc) return rc;
    if (r9) std::memcpy(r9, g->r_drift.m, sizeof(g->r_drift.m));
    if (t3) { t3[0] = g->t_drift.x; t3[1] = g->t_drift.y; t3[2] = g->t_drift.z; }
    if (yaw) *yaw = g->yaw_drift;
    return 0;
}

int vp_get_keyframe(vp_graph* g, int index, double* vio14, int* loop_index, double* loop_info8) {
    if (!g || index < 0 || index >= (int)g->kfs.size()) return VP_ERR_INVALID;
    const int rc = collect(g);
    if (rc) return rc;
    const KeyFrame& kf = g->kfs[index];
    if (vio14) {
        KeyFrame v;
        v.P = kf.vio_P;
        v.R = kf.vio_R;
        store_pose(v, vio14, vio14 + 3);
        store_pose(kf, vio14 + 7, vio14 + 10);
    }
    if (loop_index) *loop_index = kf.has_loop ? kf.loop_index : -1;
    if (loop_info8) std::memcpy(loop_info8, kf.loop_info, sizeof(kf.loop_info));
    return 0;
}

int vp_get_path(vp_graph* g, int cap, double* stamps, double* P3, double* Qwxyz, int* sequence) {
    if (!g) return VP_ERR_INVALID;
    const int rc = collect(g);
    if (rc) return rc;
    const int n = (int)g->kfs.size();
    if (cap <= 0) return n;
    if (cap < n) return VP_ERR_CAPACITY;
    for (int i = 0; i < n; i++) {
        const KeyFrame& kf = g->kfs[i];
        if (stamps) stamps[i] = kf.stamp;
        store_pose(kf, P3 ? P3 + 3 * i : nullptr, Qwxyz ? Qwxyz + 4 * i : nullptr);
        if (sequence) sequence[i] = kf.seq;
    }
    return n;
}

int vp_info(vp_graph* g, int* out8, double* costs2) {
    if (!g) return VP_ERR_INVALID;
    const int rc = collect(g);
    if (rc) return rc;
    if (out8) {
        const int v[8] = {(int)g->kfs.size(), g->n_loops, g->earliest_loop_index, g->n_opt,
                          g->last_info[0], g->last_info[1], g->last_info[2], g->last_info[3]};
        std::memcpy(out8, v, sizeof(v));
    }
    if (costs2) { costs2[0] = g->last_cost[0]; costs2[1] = g->last_cost[1]; }
    return 0;
}

int vp_last_timing(vp_graph* g, float* ms, int* launches) {
    if (!g) return VP_ERR_INVALID;
    const int rc = collect(g);
    if (rc) return rc;
    if (ms) *ms = g->last_ms;
    if (launches) *launches = g->last_launches;
    return 0;
}

int vp_save(vp_graph* g, const char* prefix) {
    if (!g || !prefix) return VP_ERR_INVALID;
    const int rc = collect(g);
    if (rc) return rc;
    std::vector<vb::MapKeyFrame> mk(g->kfs.size());
    for (size_t i = 0; i < mk.size(); i++) {
        const KeyFrame& kf = g->kfs[i];
        vb::MapKeyFrame& m = mk[i];
        m.index = (int)i;
        m.stamp = kf.stamp;
        KeyFrame v;
        v.P = kf.vio_P;
        v.R = kf.vio_R;
        store_pose(v, m.vio_T, m.vio_Q);
        store_pose(kf, m.pg_T, m.pg_Q);
        m.loop_index = kf.has_loop ? kf.loop_index : -1;
        std::memcpy(m.loop_info, kf.loop_info, sizeof(m.loop_info));
    }
    vb::LvState* lv = *vb::pg_loop_state(g->owner);
    if (lv) {
        const int r = vb::lv_read_points(lv, g->member, &mk, &g->err);
        if (r) return r;
    }
    const int w = vb::map_write(prefix, mk, lv != nullptr, &g->err);
    return w ? w : (int)mk.size();
}

int vp_load(vp_graph* g, const char* prefix) {
    if (!g || !prefix) return VP_ERR_INVALID;
    if (!g->kfs.empty()) {
        g->err = "vp_load: the graph already holds key frames; a map is loaded before the first key frame";
        return VP_ERR_INVALID;
    }
    vb::LvState* lv = *vb::pg_loop_state(g->owner);
    std::vector<vb::MapKeyFrame> mk;
    int rc = vb::map_read(prefix, lv != nullptr, g->cfg.max_keyframes, lv ? vb::lv_max_corners(lv) : 0, &mk, &g->err);
    if (rc) return rc;
    // the loaded-key-frame constructor (keyframe.cpp:44-70): the VIO pose is the saved PG pose, the rotation is
    // toRotationMatrix of the parsed quaternion as it is (not normalised)
    const int n = (int)mk.size();
    std::vector<KeyFrame> kfs(n);
    std::vector<double> P(3 * (size_t)n), Q(4 * (size_t)n);
    int earliest = -1, loops = 0;
    for (int i = 0; i < n; i++) {
        const vb::MapKeyFrame& m = mk[i];
        KeyFrame& kf = kfs[i];
        kf.stamp = m.stamp;
        kf.seq = 0;
        kf.P = kf.vio_P = Vec3(m.pg_T[0], m.pg_T[1], m.pg_T[2]);
        kf.R = kf.vio_R = Quat(m.pg_Q[0], m.pg_Q[1], m.pg_Q[2], m.pg_Q[3]).R();
        kf.has_loop = m.loop_index != -1;
        kf.loop_index = m.loop_index;
        std::memcpy(kf.loop_info, m.loop_info, sizeof(kf.loop_info));
        if (kf.has_loop) {
            loops++;
            if (earliest == -1 || m.loop_index < earliest) earliest = m.loop_index;
        }
        std::memcpy(&P[3 * (size_t)i], m.pg_T, sizeof(m.pg_T));
        std::memcpy(&Q[4 * (size_t)i], m.pg_Q, sizeof(m.pg_Q));
    }
    if (lv) {
        rc = vb::lv_write_points(lv, g->member, 0, mk, P.data(), Q.data(), &g->err);
        if (rc) return rc;
    }
    g->kfs = std::move(kfs);
    g->n_map = n;
    g->earliest_loop_index = earliest;
    g->n_loops = loops;
    return n;
}

int vp_batch_create(const vp_config* cfg, int n, vp_batch** out) {
    if (!out) return VP_ERR_INVALID;
    return batch_create(cfg, n, out);
}
void vp_batch_destroy(vp_batch* b) {
    if (b) release(b);
}
int vp_batch_size(const vp_batch* b) { return b ? b->S : VP_ERR_INVALID; }
vp_graph* vp_batch_member(vp_batch* b, int k) { return (b && k >= 0 && k < b->S) ? b->members[k] : nullptr; }
const char* vp_batch_last_error(const vp_batch* b) { return b ? b->err.c_str() : "null handle"; }
int vp_batch_optimize(vp_batch* b, const int* active, int* status) { return b ? batch_optimize(b, active, status) : VP_ERR_INVALID; }
int vp_batch_sync(vp_batch* b) {
    if (!b) return VP_ERR_INVALID;
    for (vp_graph* g : b->members) {
        const int rc = collect(g);
        if (rc) return rc;
    }
    return 0;
}
int vp_batch_last_timing(vp_batch* b, float* ms2, int* launches) {
    if (!b) return VP_ERR_INVALID;
    if (batch_wait(b)) return VP_ERR_CUDA;
    if (ms2) { ms2[0] = b->ms[0]; ms2[1] = b->ms[1]; }
    if (launches) *launches = b->launches;
    return 0;
}

int vp_debug_four_dof_error(const double* params8, const double* meas6, int weighted, int robust, double* out37) {
    if (!params8 || !meas6 || !out37) return VP_ERR_INVALID;
    if (!vb::device_available(0)) return VP_ERR_NO_DEVICE;
    vb::DeviceArray<double> d;
    if (d.alloc(8 + 6 + 37) != cudaSuccess) return VP_ERR_CUDA;
    cudaMemcpy(d, params8, sizeof(double) * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d + 8, meas6, sizeof(double) * 6, cudaMemcpyHostToDevice);
    vb::launch_pg_debug_edge(d, d + 8, weighted, robust, d + 14, nullptr);
    return cudaMemcpy(out37, d + 14, sizeof(double) * 37, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : VP_ERR_CUDA;
}

}  // extern "C"
