// Host side of loop verification (include/vinsb200/loop_verify.h): the descriptor arena a batch of pose graphs owns,
// key-frame attach and the verification of candidate pairs around the device stages of lv_kernels.cu.
#include "vinsb200/loop_verify.h"

#include "vinsb200/loop_camera.h"
#include "vinsb200/tracker.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "camera_lift.h"
#include "cuda_check.h"
#include "host_math.h"
#include "lv_kernels.h"
#include "lv_layout.h"
#include "pg_host.h"
#include "pg_map.h"

namespace vb {

static_assert((int)VP_CAMERA_PINHOLE == (int)VT_CAMERA_PINHOLE && (int)VP_CAMERA_MEI == (int)VT_CAMERA_MEI &&
                  (int)VP_CAMERA_KANNALA_BRANDT == (int)VT_CAMERA_KANNALA_BRANDT,
              "the loop-verification camera models are the tracker's");
static_assert(VP_CAMERA_PINHOLE == CAM_PINHOLE && VP_CAMERA_MEI == CAM_MEI && VP_CAMERA_KANNALA_BRANDT == CAM_KANNALA_BRANDT,
              "camera_lift.h model values");

struct LvState {
    vp_loop_config cfg{};
    int camera_model = VP_CAMERA_PINHOLE;
    double xi = 0.0;
    int pattern[4 * LV_BITS] = {};
    int S = 0, cap_kf = 0, device = 0;
    size_t slot_bytes = 0, stage_bytes = 0, conn_bytes = 0, res_doubles = 0;
    DeviceArray<char> d_arena, d_stage, d_ascratch, d_cscratch;
    PinnedArray<char> h_stage;
    DeviceArray<int> d_pattern;
    PinnedArray<int> h_status;
    PinnedArray<long long> h_jobs;
    DeviceArray<long long> d_jobs;
    PinnedArray<double> h_res;
    DeviceArray<double> d_res;
    std::vector<char> attached;  // per slot, host copy of the slot header's flag
    Stream stream;
    Event ev[8];  // 0-3 around the attach stages, 4-7 around the verification stages
    float ms[6] = {0, 0, 0, 0, 0, 0};
    ~LvState() {  // the buffers go once the stream has drained
        cudaSetDevice(device);
        if (stream) cudaStreamSynchronize(stream);
    }
};

void lv_release(LvState* s) { delete s; }

int lv_max_corners(const LvState* s) { return s->cfg.max_corners; }

int lv_read_points(LvState* s, int member, std::vector<MapKeyFrame>* kfs, std::string* err) {
    const int n = (int)kfs->size();
    if (!n) return 0;
    const LvSlotLayout sl = lv_slot_layout(s->cfg.max_window, s->cfg.max_corners);
    const char* base = s->d_arena + (size_t)member * s->cap_kf * s->slot_bytes;
    std::vector<LvSlotHdr> hdr(n);
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaSetDevice(s->device));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpy2D(hdr.data(), sizeof(LvSlotHdr), base, s->slot_bytes, sizeof(LvSlotHdr), n, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; i++) {
        MapKeyFrame& k = (*kfs)[i];
        const size_t c = s->attached[(size_t)member * s->cap_kf + i] ? (size_t)hdr[i].n_corners : 0;
        k.n_kp = (int)c;
        k.kp.resize(2 * c);
        k.kpn.resize(2 * c);
        k.desc.resize(4 * c);
        if (!c) continue;
        const char* slot = base + (size_t)i * s->slot_bytes;
        VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpy(k.kp.data(), slot + sl.kp, 8 * c, cudaMemcpyDeviceToHost));
        VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpy(k.kpn.data(), slot + sl.kpn, 8 * c, cudaMemcpyDeviceToHost));
        VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpy(k.desc.data(), slot + sl.kdesc, 32 * c, cudaMemcpyDeviceToHost));
    }
    return 0;
}

int lv_write_points(LvState* s, int member, int first, const std::vector<MapKeyFrame>& kfs, const double* P, const double* Q,
                    std::string* err) {
    const int n = (int)kfs.size();
    if (!n) return 0;
    size_t bytes = lv_load_jobs_bytes(n);
    for (const MapKeyFrame& k : kfs) bytes += lv_load_layout(k.n_kp).total;
    std::vector<char> h(bytes, 0);
    long long* jobs = reinterpret_cast<long long*>(h.data());
    size_t off = lv_load_jobs_bytes(n);
    for (int i = 0; i < n; i++) {
        const MapKeyFrame& k = kfs[i];
        const LvLoadLayout ll = lv_load_layout(k.n_kp);
        jobs[2 * i] = (long long)(((size_t)member * s->cap_kf + first + i) * s->slot_bytes);
        jobs[2 * i + 1] = (long long)off;
        LvSlotHdr hd{};
        std::memcpy(hd.vio_P, P + 3 * i, sizeof(hd.vio_P));
        std::memcpy(hd.vio_Q, Q + 4 * i, sizeof(hd.vio_Q));
        hd.n_win = 0;
        hd.n_corners = k.n_kp;
        hd.attached = 1;
        std::memcpy(h.data() + off, &hd, sizeof(hd));
        std::memcpy(h.data() + off + ll.kp, k.kp.data(), 8 * (size_t)k.n_kp);
        std::memcpy(h.data() + off + ll.kpn, k.kpn.data(), 8 * (size_t)k.n_kp);
        std::memcpy(h.data() + off + ll.kdesc, k.desc.data(), 32 * (size_t)k.n_kp);
        off += ll.total;
    }
    DeviceArray<char> d;
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaSetDevice(s->device));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, d.alloc(bytes));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpyAsync(d, h.data(), bytes, cudaMemcpyHostToDevice, s->stream));
    launch_lv_scatter(s->d_arena, d, n, s->cfg.max_window, s->cfg.max_corners, s->stream);
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaGetLastError());
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaStreamSynchronize(s->stream));
    for (int i = 0; i < n; i++) s->attached[(size_t)member * s->cap_kf + first + i] = 1;
    return 0;
}

}  // namespace vb

namespace {

using vb::LvState;

bool camera_ok(int camera_model, double xi) {
    return camera_model >= VP_CAMERA_PINHOLE && camera_model <= VP_CAMERA_KANNALA_BRANDT && std::isfinite(xi);
}

bool config_ok(const vp_loop_config* c) {
    if (!c || !c->brief_pattern || c->rows < 8 || c->rows > vb::LV_MAX_ROWS || c->cols < 8 || c->cols > vb::LV_MAX_COLS) return false;
    if (c->max_window < 1 || c->max_window > vb::LV_CAP_WINDOW || c->max_corners < 1 || c->max_corners > vb::LV_CAP_CORNERS) return false;
    if (!(c->intrinsics[0] != 0.0) || !(c->intrinsics[1] != 0.0)) return false;
    return true;
}

// The stream, events and buffers of a state whose sizes are set, on its device.
int create_resources(LvState* s, std::string* err) {
    const vp_loop_config* c = &s->cfg;
    const size_t S = (size_t)s->S;
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaSetDevice(s->device));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->stream.create());
    for (vb::Event& ev : s->ev) VB_CUDA_CHECK(err, VP_ERR_CUDA, ev.create());
    const size_t arena = vb::lv_arena_bytes(s->S, s->cap_kf, c->max_window, c->max_corners);
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->d_arena.alloc(arena));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemset(s->d_arena, 0, arena));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->d_stage.alloc(s->stage_bytes));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->h_stage.alloc(s->stage_bytes));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->d_ascratch.alloc(vb::lv_attach_layout(c->rows, c->cols).total));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->h_status.alloc(4));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->d_cscratch.alloc(S * s->conn_bytes));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemset(s->d_cscratch, 0, S * s->conn_bytes));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->d_pattern.alloc(4 * vb::LV_BITS));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpy(s->d_pattern, s->pattern, sizeof(s->pattern), cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->d_jobs.alloc(S * 2));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->h_jobs.alloc(S * 2));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->d_res.alloc(S * s->res_doubles));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, s->h_res.alloc(S * s->res_doubles));
    return 0;
}

int enable(LvState** slot, const vp_loop_config* c, int camera_model, double xi, int S, int cap_kf, int device, std::string* err) {
    if (!config_ok(c) || !camera_ok(camera_model, xi)) {
        *err = "vp_loop_enable: invalid configuration";
        return VP_ERR_INVALID;
    }
    if (*slot) {
        *err = "vp_loop_enable: loop verification is already enabled";
        return VP_ERR_INVALID;
    }
    std::unique_ptr<LvState> s(new LvState);
    s->cfg = *c;
    s->cfg.brief_pattern = nullptr;
    s->camera_model = camera_model;
    s->xi = xi;
    std::memcpy(s->pattern, c->brief_pattern, sizeof(s->pattern));
    s->S = S;
    s->cap_kf = cap_kf;
    s->device = device;
    s->slot_bytes = vb::lv_slot_layout(c->max_window, c->max_corners).total;
    s->stage_bytes = vb::lv_stage_layout(c->rows, c->cols, c->max_window).total;
    s->conn_bytes = vb::lv_conn_layout(c->max_window).total;
    s->res_doubles = vb::lv_result_doubles(c->max_window);
    s->attached.assign((size_t)S * cap_kf, 0);
    const int rc = create_resources(s.get(), err);
    // the failure is also the thread's last CUDA error: cleared here; an allocation that does not fit is a capacity error
    if (rc) return cudaGetLastError() == cudaErrorMemoryAllocation ? VP_ERR_CAPACITY : rc;
    *slot = s.release();
    return 0;
}

// After a failed call the stream may hold part of a launch chain: it is drained so that the next call starts clean.
int drain_on_error(LvState* s, int rc) {
    if (rc) {
        cudaStreamSynchronize(s->stream);
        cudaGetLastError();
    }
    return rc;
}

// One staged key frame into arena slot `slot`: the input copy, the attach chain, the status copy, then a wait.
int attach_chain(LvState* s, size_t slot, std::string* err) {
    const vp_loop_config& c = s->cfg;
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaSetDevice(s->device));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpyAsync(s->d_stage, s->h_stage, s->stage_bytes, cudaMemcpyHostToDevice, s->stream));
    vb::LvAttachLaunch L{s->d_stage, s->d_ascratch, s->d_arena + slot * s->slot_bytes, s->d_pattern,
                         c.rows, c.cols, c.max_window, c.max_corners, {}, s->camera_model, s->xi};
    std::memcpy(L.intrinsics, c.intrinsics, sizeof(L.intrinsics));
    cudaEvent_t ev[4] = {s->ev[0], s->ev[1], s->ev[2], s->ev[3]};
    vb::launch_lv_attach(L, s->stream, ev);
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaGetLastError());
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpyAsync(s->h_status, s->d_ascratch + vb::lv_attach_layout(c.rows, c.cols).status, 8,
                                                    cudaMemcpyDeviceToHost, s->stream));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaStreamSynchronize(s->stream));
    for (int k = 0; k < 3; k++) cudaEventElapsedTime(&s->ms[k], s->ev[k], s->ev[k + 1]);
    return 0;
}

int attach(LvState* s, int member, int index, const double* P3, const double* Q4, const uint8_t* img, size_t stride, int n,
           const float* p3d, const float* uv, const float* norm, const double* ids, int* n_corners, std::string* err) {
    const vp_loop_config& c = s->cfg;
    if (index < 0 || index >= s->cap_kf || !P3 || !Q4 || !img || stride < (size_t)c.cols || n < 0 ||
        (n > 0 && (!p3d || !uv || !norm || !ids))) {
        *err = "vp_attach_keyframe: invalid argument";
        return VP_ERR_INVALID;
    }
    if (n > c.max_window) {
        *err = "vp_attach_keyframe: " + std::to_string(n) + " window points, at most max_window = " + std::to_string(c.max_window);
        return VP_ERR_CAPACITY;
    }
    const vb::LvStageLayout st = vb::lv_stage_layout(c.rows, c.cols, c.max_window);
    vb::LvSlotHdr h{};
    std::memcpy(h.vio_P, P3, sizeof(h.vio_P));
    std::memcpy(h.vio_Q, Q4, sizeof(h.vio_Q));
    h.n_win = n;
    std::memcpy(s->h_stage, &h, sizeof(h));
    for (int y = 0; y < c.rows; y++) std::memcpy(s->h_stage + st.img + (size_t)y * c.cols, img + (size_t)y * stride, c.cols);
    if (n) {
        std::memcpy(s->h_stage + st.p3d, p3d, 12 * (size_t)n);
        std::memcpy(s->h_stage + st.uv, uv, 8 * (size_t)n);
        std::memcpy(s->h_stage + st.norm, norm, 8 * (size_t)n);
        std::memcpy(s->h_stage + st.id, ids, 8 * (size_t)n);
    }
    const int rc = drain_on_error(s, attach_chain(s, (size_t)member * s->cap_kf + index, err));
    if (rc) return rc;
    if (n_corners) *n_corners = s->h_status[0];
    if (s->h_status[1]) {
        *err = "vp_attach_keyframe: " + std::to_string(s->h_status[0]) + " FAST corners, at most max_corners = " + std::to_string(c.max_corners);
        return VP_ERR_CAPACITY;
    }
    s->attached[(size_t)member * s->cap_kf + index] = 1;
    return 0;
}

// The job copy, the verification chain of `jobs` pairs, the result copy, then a wait.
int connect_chain(LvState* s, int jobs, int match, std::string* err) {
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaSetDevice(s->device));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpyAsync(s->d_jobs, s->h_jobs, (size_t)jobs * 2 * sizeof(long long), cudaMemcpyHostToDevice, s->stream));
    vb::LvConnLaunch L{s->d_arena, s->d_jobs, s->d_cscratch, s->conn_bytes, s->d_res, s->res_doubles, jobs, s->cfg.max_window,
                       s->cfg.max_corners, {}, {}};
    std::memcpy(L.ric, s->cfg.ric9, sizeof(L.ric));
    std::memcpy(L.tic, s->cfg.tic3, sizeof(L.tic));
    cudaEvent_t ev[4] = {s->ev[4], s->ev[5], s->ev[6], s->ev[7]};
    vb::launch_lv_connect(L, s->stream, ev, match);
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaGetLastError());
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaMemcpyAsync(s->h_res, s->d_res, (size_t)jobs * s->res_doubles * sizeof(double),
                                                    cudaMemcpyDeviceToHost, s->stream));
    VB_CUDA_CHECK(err, VP_ERR_CUDA, cudaStreamSynchronize(s->stream));
    for (int k = 0; k < 3; k++) cudaEventElapsedTime(&s->ms[3 + k], s->ev[4 + k], s->ev[5 + k]);
    return 0;
}

// Verifies the pairs of the members with cur[k] >= 0 in one launch chain; match = 0 keeps the match lists already in
// the scratch (the PnP test entry).
int connect(LvState* s, const int* cur, const int* old, vp_loop_result* r, int cap, double* xyid, int* status, std::string* err,
            int match = 1) {
    int jobs = 0;
    std::vector<int> member;
    for (int k = 0; k < s->S; k++) {
        if (status) status[k] = 0;
        if (cur[k] < 0) continue;
        const size_t base = (size_t)k * s->cap_kf;
        if (cur[k] >= s->cap_kf || old[k] < 0 || old[k] >= s->cap_kf || cur[k] == old[k] || !s->attached[base + cur[k]] ||
            !s->attached[base + old[k]]) {
            *err = "vp_find_connection: cur and old must be two different attached key frames";
            if (status) status[k] = VP_ERR_INVALID;
            return VP_ERR_INVALID;
        }
        s->h_jobs[2 * jobs] = (long long)((base + cur[k]) * s->slot_bytes);
        s->h_jobs[2 * jobs + 1] = (long long)((base + old[k]) * s->slot_bytes);
        member.push_back(k);
        jobs++;
    }
    if (!jobs) return 0;
    const int rc = drain_on_error(s, connect_chain(s, jobs, match, err));
    if (rc) return rc;
    for (int j = 0; j < jobs; j++) {
        const int k = member[j];
        const double* o = s->h_res + (size_t)j * s->res_doubles;
        vp_loop_result& rr = r[k];
        rr.accepted = (int)o[0];
        rr.n_matches = (int)o[1];
        rr.n_inliers = (int)o[2];
        const int np = (int)o[3];
        rr.n_points = xyid ? (np < cap ? np : cap) : 0;
        for (int i = 0; i < 3; i++) rr.loop_info[i] = o[vb::LV_RES_LOOP + i];
        rr.loop_info[7] = o[vb::LV_RES_LOOP + 7];
        hm::Mat3 rq;
        for (int i = 0; i < 9; i++) rq(i / 3, i % 3) = o[vb::LV_RES_RQ + i];
        const hm::Quat q = rr.n_inliers ? hm::Quat::FromR(rq) : hm::Quat(1, 0, 0, 0);
        rr.loop_info[3] = q.w;
        rr.loop_info[4] = q.x;
        rr.loop_info[5] = q.y;
        rr.loop_info[6] = q.z;
        std::memcpy(rr.old_R9, o + vb::LV_RES_R, sizeof(rr.old_R9));
        std::memcpy(rr.old_T3, o + vb::LV_RES_T, sizeof(rr.old_T3));
        if (rr.n_points) std::memcpy(xyid + 3 * (size_t)cap * k, o + vb::LV_RES_LIST, 3 * sizeof(double) * rr.n_points);
        if (status) status[k] = 1;
    }
    return 0;
}

// A batch-of-one state for the vp_debug_* entries: key frames 0 (cur) and 1 (old) of one graph, device 0.
struct DebugState {
    LvState* s = nullptr;
    std::string err;
    int rc = 0;
    DebugState(int rows, int cols, const int* pattern, int max_window, int max_corners) {
        if (!vb::device_available(0)) {
            rc = VP_ERR_NO_DEVICE;
            return;
        }
        static const int zero_pattern[4 * vb::LV_BITS] = {};
        vp_loop_config c{};
        c.rows = rows;
        c.cols = cols;
        c.intrinsics[0] = c.intrinsics[1] = 1.0;
        c.ric9[0] = c.ric9[4] = c.ric9[8] = 1.0;
        c.brief_pattern = pattern ? pattern : zero_pattern;
        c.max_window = max_window;
        c.max_corners = max_corners;
        rc = enable(&s, &c, VP_CAMERA_PINHOLE, 0.0, 1, 2, 0, &err);
    }
    ~DebugState() { vb::lv_release(s); }
    char* slot(int k) const { return s->d_arena + k * s->slot_bytes; }
};

const double kIdentityQ[4] = {1, 0, 0, 0}, kZeroP[3] = {0, 0, 0};

}  // namespace

extern "C" {

int vp_loop_enable(vp_graph* g, const vp_loop_config* cfg) { return vp_loop_enable_camera(g, cfg, VP_CAMERA_PINHOLE, 0.0); }

int vp_batch_loop_enable(vp_batch* b, const vp_loop_config* cfg) { return vp_batch_loop_enable_camera(b, cfg, VP_CAMERA_PINHOLE, 0.0); }

int vp_loop_enable_camera(vp_graph* g, const vp_loop_config* cfg, int camera_model, double xi) {
    if (!g) return VP_ERR_INVALID;
    int member = 0, device = 0;
    bool standalone = false;
    vp_batch* b = vb::pg_owner(g, &member, &standalone);
    if (!standalone) {
        *vb::pg_error(g) = "vp_loop_enable: a batch member is enabled through vp_batch_loop_enable";
        return VP_ERR_INVALID;
    }
    const int cap = vb::pg_capacity(b, &device);
    return enable(vb::pg_loop_state(b), cfg, camera_model, xi, 1, cap, device, vb::pg_error(g));
}

int vp_batch_loop_enable_camera(vp_batch* b, const vp_loop_config* cfg, int camera_model, double xi) {
    if (!b) return VP_ERR_INVALID;
    int device = 0;
    const int cap = vb::pg_capacity(b, &device);
    return enable(vb::pg_loop_state(b), cfg, camera_model, xi, vp_batch_size(b), cap, device, vb::pg_batch_error(b));
}

int vp_attach_keyframe(vp_graph* g, int index, const double* vio_P3, const double* vio_Qwxyz, const uint8_t* img, size_t row_stride,
                       int n, const float* point_3d, const float* point_uv, const float* point_norm, const double* point_id,
                       int* n_corners) {
    if (!g) return VP_ERR_INVALID;
    int member = 0;
    bool standalone = false;
    LvState* s = *vb::pg_loop_state(vb::pg_owner(g, &member, &standalone));
    if (!s) {
        *vb::pg_error(g) = "vp_attach_keyframe: loop verification is not enabled";
        return VP_ERR_INVALID;
    }
    return attach(s, member, index, vio_P3, vio_Qwxyz, img, row_stride, n, point_3d, point_uv, point_norm, point_id, n_corners,
                  vb::pg_error(g));
}

int vp_find_connection(vp_graph* g, int cur, int old, vp_loop_result* r, int cap, double* match_xyid) {
    if (!g || !r || (match_xyid && cap < 0)) return VP_ERR_INVALID;
    int member = 0;
    bool standalone = false;
    LvState* s = *vb::pg_loop_state(vb::pg_owner(g, &member, &standalone));
    if (!s) {
        *vb::pg_error(g) = "vp_find_connection: loop verification is not enabled";
        return VP_ERR_INVALID;
    }
    std::vector<int> c(s->S, -1), o(s->S, -1);
    std::vector<vp_loop_result> rr(s->S);
    c[member] = cur < 0 ? s->cap_kf : cur;  // a negative index is an argument error here, not "skip"
    o[member] = old;
    std::vector<double> list;
    if (match_xyid) list.assign((size_t)3 * cap * s->S, 0.0);
    const int rc = connect(s, c.data(), o.data(), rr.data(), cap, match_xyid ? list.data() : nullptr, nullptr, vb::pg_error(g));
    if (rc) return rc;
    *r = rr[member];
    if (match_xyid && r->n_points) std::memcpy(match_xyid, list.data() + 3 * (size_t)cap * member, 3 * sizeof(double) * r->n_points);
    return r->accepted;
}

int vp_batch_find_connection(vp_batch* b, const int* cur, const int* old, vp_loop_result* r, int cap, double* match_xyid, int* status) {
    if (!b || !cur || !old || !r || (match_xyid && cap < 0)) return VP_ERR_INVALID;
    LvState* s = *vb::pg_loop_state(b);
    if (!s) {
        *vb::pg_batch_error(b) = "vp_batch_find_connection: loop verification is not enabled";
        return VP_ERR_INVALID;
    }
    return connect(s, cur, old, r, cap, match_xyid, status, vb::pg_batch_error(b));
}

int vp_loop_last_timing(vp_graph* g, float* ms6) {
    if (!g || !ms6) return VP_ERR_INVALID;
    int member = 0;
    bool standalone = false;
    LvState* s = *vb::pg_loop_state(vb::pg_owner(g, &member, &standalone));
    if (!s) return VP_ERR_INVALID;
    std::memcpy(ms6, s->ms, sizeof(s->ms));
    return 0;
}

int vp_batch_loop_last_timing(vp_batch* b, float* ms6) {
    if (!b || !ms6 || !*vb::pg_loop_state(b)) return VP_ERR_INVALID;
    std::memcpy(ms6, (*vb::pg_loop_state(b))->ms, sizeof(float) * 6);
    return 0;
}

int vp_debug_brief_blur(const uint8_t* img, int rows, int cols, uint8_t* out) {
    if (!img || !out) return VP_ERR_INVALID;
    DebugState d(rows, cols, nullptr, 1, vb::LV_CAP_CORNERS);
    if (d.rc) return d.rc;
    int nc = 0;
    int rc = attach(d.s, 0, 0, kZeroP, kIdentityQ, img, cols, 0, nullptr, nullptr, nullptr, nullptr, &nc, &d.err);
    if (rc && rc != VP_ERR_CAPACITY) return rc;
    return cudaMemcpy(out, d.s->d_ascratch + vb::lv_attach_layout(rows, cols).blur, (size_t)rows * cols, cudaMemcpyDeviceToHost) == cudaSuccess
               ? 0 : VP_ERR_CUDA;
}

int vp_debug_fast(const uint8_t* img, int rows, int cols, int cap, float* xy) {
    if (!img || !xy || cap < 1 || cap > vb::LV_CAP_CORNERS) return VP_ERR_INVALID;
    DebugState d(rows, cols, nullptr, 1, cap);
    if (d.rc) return d.rc;
    int nc = 0;
    const int rc = attach(d.s, 0, 0, kZeroP, kIdentityQ, img, cols, 0, nullptr, nullptr, nullptr, nullptr, &nc, &d.err);
    if (rc) return rc;
    const size_t off = vb::lv_slot_layout(1, cap).kp;
    return cudaMemcpy(xy, d.slot(0) + off, 8 * (size_t)nc, cudaMemcpyDeviceToHost) == cudaSuccess ? nc : VP_ERR_CUDA;
}

int vp_debug_brief(const uint8_t* img, int rows, int cols, const int* pattern, int n, const float* uv, uint64_t* desc) {
    if (!img || !pattern || !uv || !desc || n < 1 || n > vb::LV_CAP_WINDOW) return VP_ERR_INVALID;
    DebugState d(rows, cols, pattern, n, vb::LV_CAP_CORNERS);
    if (d.rc) return d.rc;
    std::vector<float> zeros(3 * (size_t)n, 0.f);
    std::vector<double> ids(n, 0.0);
    int nc = 0;
    const int rc = attach(d.s, 0, 0, kZeroP, kIdentityQ, img, cols, n, zeros.data(), uv, zeros.data(), ids.data(), &nc, &d.err);
    if (rc) return rc;
    const size_t off = vb::lv_slot_layout(n, vb::LV_CAP_CORNERS).wdesc;
    return cudaMemcpy(desc, d.slot(0) + off, 32 * (size_t)n, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : VP_ERR_CUDA;
}

int vp_debug_match(int na, const uint64_t* a, int nb, const uint64_t* b, int* idx) {
    if (!a || !idx || na < 1 || na > vb::LV_CAP_WINDOW || nb < 0 || nb > vb::LV_CAP_CORNERS || (nb && !b)) return VP_ERR_INVALID;
    DebugState d(8, 8, nullptr, na, nb ? nb : 1);
    if (d.rc) return d.rc;
    const vb::LvSlotLayout sl = vb::lv_slot_layout(na, nb ? nb : 1);
    vb::LvSlotHdr h0{}, h1{};
    h0.n_win = na;
    h0.vio_Q[0] = h1.vio_Q[0] = 1;
    h1.n_corners = nb;
    h0.attached = h1.attached = 1;
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(0), &h0, sizeof(h0), cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(1), &h1, sizeof(h1), cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(0) + sl.wdesc, a, 32 * (size_t)na, cudaMemcpyHostToDevice));
    if (nb) VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(1) + sl.kdesc, b, 32 * (size_t)nb, cudaMemcpyHostToDevice));
    d.s->attached[0] = d.s->attached[1] = 1;
    const int cur = 0, old = 1;
    vp_loop_result r{};
    const int rc = connect(d.s, &cur, &old, &r, 0, nullptr, nullptr, &d.err);
    if (rc) return rc;
    return cudaMemcpy(idx, d.s->d_cscratch + vb::lv_conn_layout(na).win_match, 4 * (size_t)na, cudaMemcpyDeviceToHost) == cudaSuccess
               ? 0 : VP_ERR_CUDA;
}

int vp_debug_pnp(int n, const float* point_3d, const float* norm, double* Rt12, int* n_inliers, uint8_t* inlier) {
    if (!point_3d || !norm || !Rt12 || n <= vb::LV_MIN_LOOP_NUM || n > vb::LV_CAP_WINDOW) return VP_ERR_INVALID;
    DebugState d(8, 8, nullptr, n, n);
    if (d.rc) return d.rc;
    const vb::LvSlotLayout sl = vb::lv_slot_layout(n, n);
    const vb::LvConnLayout cl = vb::lv_conn_layout(n);
    vb::LvSlotHdr h0{}, h1{};
    h0.n_win = n;
    h0.vio_Q[0] = h1.vio_Q[0] = 1;
    h1.n_corners = n;
    h0.attached = h1.attached = 1;
    std::vector<double> ids(n);
    std::vector<int> iota(n);
    for (int i = 0; i < n; i++) ids[i] = iota[i] = i;
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(0), &h0, sizeof(h0), cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(1), &h1, sizeof(h1), cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(0) + sl.p3d, point_3d, 12 * (size_t)n, cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(0) + sl.id, ids.data(), 8 * (size_t)n, cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.slot(1) + sl.kpn, norm, 8 * (size_t)n, cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.s->d_cscratch, &n, sizeof(int), cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.s->d_cscratch + cl.win_match, iota.data(), 4 * (size_t)n, cudaMemcpyHostToDevice));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpy(d.s->d_cscratch + cl.midx, iota.data(), 4 * (size_t)n, cudaMemcpyHostToDevice));
    d.s->attached[0] = d.s->attached[1] = 1;
    const int cur = 0, old = 1;
    vp_loop_result r{};
    std::vector<double> list(3 * (size_t)n);
    const int rc = connect(d.s, &cur, &old, &r, n, list.data(), nullptr, &d.err, 0);
    if (rc) return rc;
    // with an identity current pose and extrinsic, PnP_R_old = R^T and PnP_T_old = -R^T t
    for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++) Rt12[3 * a + b] = r.old_R9[3 * b + a];
    }
    for (int a = 0; a < 3; a++) Rt12[9 + a] = -(Rt12[3 * a] * r.old_T3[0] + Rt12[3 * a + 1] * r.old_T3[1] + Rt12[3 * a + 2] * r.old_T3[2]);
    if (n_inliers) *n_inliers = r.n_inliers;
    if (inlier) {
        std::memset(inlier, 0, n);
        for (int i = 0; i < r.n_points; i++) inlier[(int)list[3 * i + 2]] = 1;
    }
    return 0;
}

int vp_debug_lift(int camera_model, const double* intrinsics8, double xi, int n, const float* uv, float* xy) {
    if (!intrinsics8 || !uv || !xy || n < 1 || n > vb::LV_CAP_CORNERS || !camera_ok(camera_model, xi) || !(intrinsics8[0] != 0.0) ||
        !(intrinsics8[1] != 0.0))
        return VP_ERR_INVALID;
    DebugState d(8, 8, nullptr, 1, n);
    if (d.rc) return d.rc;
    LvState* s = d.s;
    const vb::LvSlotLayout sl = vb::lv_slot_layout(1, n);
    const int status[2] = {n, 0};
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpyAsync(d.slot(0) + sl.kp, uv, 8 * (size_t)n, cudaMemcpyHostToDevice, s->stream));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpyAsync(s->d_ascratch + vb::lv_attach_layout(8, 8).status, status, sizeof(status),
                                                      cudaMemcpyHostToDevice, s->stream));
    vb::LvAttachLaunch L{s->d_stage, s->d_ascratch, d.slot(0), s->d_pattern, 8, 8, 1, n, {}, camera_model, xi};
    std::memcpy(L.intrinsics, intrinsics8, sizeof(L.intrinsics));
    vb::launch_lv_lift(L, s->stream);
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaGetLastError());
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaMemcpyAsync(xy, d.slot(0) + sl.kpn, 8 * (size_t)n, cudaMemcpyDeviceToHost, s->stream));
    VB_CUDA_CHECK(&d.err, VP_ERR_CUDA, cudaStreamSynchronize(s->stream));
    return 0;
}

}  // extern "C"
