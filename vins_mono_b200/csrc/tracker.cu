// vt_* C ABI: the feature-tracker pipeline (FeatureTracker::readImage and img_callback of the reference,
// feature_tracker/src/feature_tracker.cpp:81-306, feature_tracker_node.cpp:28-165) driven from the host with
// every image-sized operation on the GPU.
//
// Execution model: trackers are members of a batch (vt_batch; a stand-alone handle is a batch of one) that advance
// image by image together.  Per image step:
//   prepare (host, per member)  ->  one H2D copy (descriptors, points[, frames])  ->  CLAHE (2 kernels), pyramid (3), LK (1,
//   all points, all levels, inBorder cull fused) for ALL members, member = last grid dimension  ->  one D2H copy
//   (points + status)  ->  host: compaction; on publishing frames F-RANSAC + setMask bookkeeping (<= max_cnt points)
//   ->  one H2D copy (disc centres)  ->  mask, Shi-Tomasi map + masked max, candidates, sort, greedy select for all
//   publishing members  ->  one D2H copy (new corners)  ->  host: addPoints, undistortedPoints, updateID.
// Images, pyramids, masks and all scratch stay resident in HBM; only O(max_cnt) point data crosses PCIe (plus the frame
// itself when it is given as a host pointer).
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "batch_host.h"
#include "fe_kernels.h"
#include "fm_ransac.h"
#include "hostpool.h"
#include "kprof.h"
#include "camera_lift.h"
#include "cuda_check.h"
#include "vinsb200/tracker.h"

namespace {

struct Pt {
    float x, y;
};

struct DevicePyramid {
    vb::DeviceArray<uint8_t> base;
    vb::PyramidView view{};
};

inline int cv_round(float v) { return (int)lrintf(v); }

// The batch's point arenas (byte offsets), S members of `cap` points each.  up, host to device: pts_in (S x cap x 2 f32)
// | centres (S x cap x 2 i32).  down, device to host: pts_out (S x cap x 2 f32) | status (S x cap) | counts (S x
// FE_COUNT_SLOT i32, 16-byte aligned) | new_pts (S x cap x 2 f32).  The tracking part of each arena comes first, so a
// frame copies only what its phases produced.
struct ArenaLayout {
    size_t cap;
    size_t centres, up_bytes;                              // up arena; pts_in at 0
    size_t status, track_bytes, counts, new_pts, dn_bytes;  // down arena; pts_out at 0
};
ArenaLayout arena_layout(size_t S, size_t cap) {
    ArenaLayout a{};
    a.cap = cap;
    a.centres = S * cap * 2 * sizeof(float);
    a.up_bytes = a.centres + S * cap * 2 * sizeof(int);
    a.status = S * cap * 2 * sizeof(float);
    a.track_bytes = a.status + S * cap;
    a.counts = (a.track_bytes + 15) & ~(size_t)15;
    a.new_pts = a.counts + S * vb::FE_COUNT_SLOT * sizeof(int);
    a.dn_bytes = a.new_pts + S * cap * 2 * sizeof(float);
    return a;
}
struct ArenaSlots {  // one member's slots in the arenas at one pair of base addresses (pinned host or device)
    float* pts_in;
    int* centres;
    float* pts_out;
    uint8_t* status;
    int* counts;
    float* new_pts;
};
ArenaSlots arena_slots(const ArenaLayout& a, uint8_t* up, uint8_t* dn, int k) {
    const size_t cap = a.cap;
    ArenaSlots s;
    s.pts_in = reinterpret_cast<float*>(up) + k * cap * 2;
    s.centres = reinterpret_cast<int*>(up + a.centres) + k * cap * 2;
    s.pts_out = reinterpret_cast<float*>(dn) + k * cap * 2;
    s.status = dn + a.status + k * cap;
    s.counts = reinterpret_cast<int*>(dn + a.counts) + (size_t)k * vb::FE_COUNT_SLOT;
    s.new_pts = reinterpret_cast<float*>(dn + a.new_pts) + k * cap * 2;
    return s;
}

}  // namespace

struct vt_tracker : vb::MemberBase<vt_batch> {
    vt_config cfg{};
    // device memory of this member
    vb::DeviceArray<uint8_t> d_lut;
    DevicePyramid pyr[2];
    int cur = 0;  // pyr[cur] = cur_img pyramid, pyr[cur^1] = forw_img pyramid
    vb::DeviceArray<uint8_t> d_mask;
    vb::DeviceArray<uint8_t> d_fisheye;
    std::vector<uint8_t> owned_fisheye_mask;  // host copy read by setMask
    vb::DeviceArray<float> d_eig;
    vb::DeviceArray<unsigned long long> d_keys;
    int key_capacity = 0;
    vb::DeviceArray<int> d_cell_cnt;
    vb::DeviceArray<short2> d_cell_pts;
    // this member's slots in the batch arenas
    uint8_t* d_raw = nullptr;  // frame slot (host-image path)
    uint8_t* h_img = nullptr;
    ArenaSlots h{}, d{};  // in the pinned arenas and in their device copies
    std::vector<int> halfw;
    int capacity = 0;
    // FeatureTracker state (feature_tracker.h:45-64)
    bool have_img = false;
    std::vector<Pt> cur_pts, forw_pts, cur_un_pts, pts_velocity, n_pts;
    std::vector<int> ids, track_cnt;
    std::map<int, Pt> cur_un_pts_map, prev_un_pts_map;
    double cur_time = 0, prev_time = 0;
    int n_id = 0;
    // img_callback state (feature_tracker_node.cpp:21-26)
    double first_image_time = 0, last_image_time = 0;
    int pub_count = 1;
    bool first_image_flag = true, init_pub = false;
    // the current image step
    int status = VT_OK;
    bool step_active = false, step_pub = false, step_first = false, step_detect = false;
    int step_n = 0, step_kept = 0, step_max_new = 0;
    size_t h2d_bytes = 0, d2h_bytes = 0;
    double host_ms_ransac = 0, host_ms_mask = 0;
};

struct vt_batch : vb::BatchBase<vt_tracker> {
    vt_config cfg{};
    vb::Stream stream;
    vb::Event ev0, ev1;
    vb::PinnedArray<vb::FeSeq> h_seq;
    vb::DeviceArray<vb::FeSeq> d_seq;
    int raw_pitch = 0, capacity = 0, nlev = 0;
    vb::DeviceArray<uint8_t> d_raw;   // S x rows x raw_pitch
    vb::PinnedArray<uint8_t> h_img;   // S x rows x cols
    ArenaLayout ar{};
    vb::PinnedArray<uint8_t> h_up;    // up arena
    vb::DeviceArray<uint8_t> d_up;
    vb::PinnedArray<uint8_t> h_dn;    // down arena
    vb::DeviceArray<uint8_t> d_dn;
    vb::DeviceArray<int> d_halfw;
    vb::KernelProfile prof;  // 0 clahe_lut+apply, 1 pyrdown x3, 2 lk, 3 mask, 4 min_eig, 5 candidates+sort+select
    std::unique_ptr<vb::HostPool> pool;
    float last_ms = 0;
    int last_launches = 0;
};

namespace {

int align_up(int v, int a) { return (v + a - 1) / a * a; }

int lk_levels(int rows, int cols, int win, int max_level) {
    int lv = 0, r = rows, c = cols;
    while (lv < max_level) {
        const int nr = (r + 1) / 2, nc = (c + 1) / 2;
        if (nc <= win || nr <= win) break;
        r = nr;
        c = nc;
        lv++;
    }
    return lv;
}

cudaError_t alloc_pyramid(const vt_tracker* t, DevicePyramid& p) {
    const int nlev = lk_levels(t->cfg.rows, t->cfg.cols, 21, 3);
    size_t total = 0, offs[vb::MAX_PYR_LEVELS];
    int r = t->cfg.rows, c = t->cfg.cols;
    for (int l = 0; l <= nlev; l++) {
        p.view.rows[l] = r;
        p.view.cols[l] = c;
        p.view.pitch[l] = align_up(c, 64);
        offs[l] = total;
        total += (size_t)align_up(p.view.pitch[l] * r, 256);
        r = (r + 1) / 2;
        c = (c + 1) / 2;
    }
    p.view.nlev = nlev;
    const cudaError_t e = p.base.alloc(total);
    for (int l = 0; l <= nlev; l++) p.view.img[l] = p.base + offs[l];
    for (int l = nlev + 1; l < vb::MAX_PYR_LEVELS; l++) p.view.img[l] = nullptr;
    return e;
}

// Half widths of cv::circle(..., FILLED) per row offset (midpoint algorithm of OpenCV's Circle()).
std::vector<int> disc_half_widths(int radius) {
    std::vector<int> hw(radius + 1, -1);
    int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
    while (dx >= dy) {
        hw[dy] = std::max(hw[dy], dx);  // rows cy +- dy span cx +- dx
        hw[dx] = std::max(hw[dx], dy);  // rows cy +- dx span cx +- dy
        dy++;
        err += plus;
        plus += 2;
        const int mask = (err <= 0) - 1;
        err -= minus & mask;
        dx += mask;
        minus -= mask & 2;
    }
    return hw;
}

// CameraPtr::liftProjective followed by the division by z that every caller applies (feature_tracker.cpp:179-186, 268-272);
// camera_lift.h holds the three models.
static_assert(VT_CAMERA_PINHOLE == vb::CAM_PINHOLE && VT_CAMERA_MEI == vb::CAM_MEI && VT_CAMERA_KANNALA_BRANDT == vb::CAM_KANNALA_BRANDT,
              "camera model values");
void lift_projective(const vt_config& c, double px, double py, double& X, double& Y) {
    vb::lift_projective(c.camera_model, c.intrinsics, c.xi, px, py, X, Y);
}

template <class T>
void compact(std::vector<T>& v, const uint8_t* keep) {
    size_t j = 0;
    for (size_t i = 0; i < v.size(); i++)
        if (keep[i]) v[j++] = v[i];
    v.resize(j);
}

// rejectWithF (feature_tracker.cpp:169-202)
void reject_with_f(vt_tracker* t) {
    const int n = (int)t->forw_pts.size();
    if (n < 8) return;
    std::vector<float> a(2 * n), b(2 * n);
    const double f = t->cfg.focal_length, cx = t->cfg.cols / 2.0, cy = t->cfg.rows / 2.0;
    for (int i = 0; i < n; i++) {
        double X, Y;
        lift_projective(t->cfg, t->cur_pts[i].x, t->cur_pts[i].y, X, Y);
        a[2 * i] = (float)(f * X / 1.0 + cx);
        a[2 * i + 1] = (float)(f * Y / 1.0 + cy);
        lift_projective(t->cfg, t->forw_pts[i].x, t->forw_pts[i].y, X, Y);
        b[2 * i] = (float)(f * X / 1.0 + cx);
        b[2 * i + 1] = (float)(f * Y / 1.0 + cy);
    }
    std::vector<uint8_t> status(n);
    vb::fundamental_ransac_mask(a.data(), b.data(), n, t->cfg.f_threshold, 0.99, status.data());
    compact(t->cur_pts, status.data());
    compact(t->forw_pts, status.data());
    compact(t->cur_un_pts, status.data());
    compact(t->ids, status.data());
    compact(t->track_cnt, status.data());
}

// setMask (feature_tracker.cpp:36-69): same std::sort call (unstable, libstdc++ introsort) on the same
// element type layout; the "is the mask still 255 here" test is evaluated against the discs already
// drawn instead of a rasterised image.  Produces the integer disc centres for the device mask.
int set_mask(vt_tracker* t) {
    std::vector<std::pair<int, std::pair<Pt, int>>> cnt_pts_id;
    for (size_t i = 0; i < t->forw_pts.size(); i++)
        cnt_pts_id.push_back(std::make_pair(t->track_cnt[i], std::make_pair(t->forw_pts[i], t->ids[i])));
    std::sort(cnt_pts_id.begin(), cnt_pts_id.end(),
              [](const std::pair<int, std::pair<Pt, int>>& a, const std::pair<int, std::pair<Pt, int>>& b) {
                  return a.first > b.first;
              });
    t->forw_pts.clear();
    t->ids.clear();
    t->track_cnt.clear();
    const int r = t->cfg.min_dist;
    int kept = 0;
    for (auto& it : cnt_pts_id) {
        const int px = cv_round(it.second.first.x), py = cv_round(it.second.first.y);
        bool free_px = true;
        if (t->cfg.fisheye && t->cfg.fisheye_mask) free_px = t->cfg.fisheye_mask[(size_t)py * t->cfg.cols + px] == 255;
        for (int k = 0; k < kept && free_px; k++) {
            const int dy = std::abs(py - t->h.centres[2 * k + 1]), dx = std::abs(px - t->h.centres[2 * k]);
            if (dy <= r && dx <= t->halfw[dy]) free_px = false;
        }
        if (free_px) {
            t->forw_pts.push_back(it.second.first);
            t->ids.push_back(it.second.second);
            t->track_cnt.push_back(it.first);
            t->h.centres[2 * kept] = px;
            t->h.centres[2 * kept + 1] = py;
            kept++;
        }
    }
    return kept;
}

// undistortedPoints (feature_tracker.cpp:258-306)
void undistorted_points(vt_tracker* t) {
    t->cur_un_pts.clear();
    t->cur_un_pts_map.clear();
    for (size_t i = 0; i < t->cur_pts.size(); i++) {
        double X, Y;
        lift_projective(t->cfg, t->cur_pts[i].x, t->cur_pts[i].y, X, Y);
        const Pt u{(float)(X / 1.0), (float)(Y / 1.0)};
        t->cur_un_pts.push_back(u);
        t->cur_un_pts_map.insert(std::make_pair(t->ids[i], u));
    }
    if (!t->prev_un_pts_map.empty()) {
        const double dt = t->cur_time - t->prev_time;
        t->pts_velocity.clear();
        for (size_t i = 0; i < t->cur_un_pts.size(); i++) {
            Pt v{0, 0};
            if (t->ids[i] != -1) {
                auto it = t->prev_un_pts_map.find(t->ids[i]);
                if (it != t->prev_un_pts_map.end())
                    v = Pt{(float)((t->cur_un_pts[i].x - it->second.x) / dt), (float)((t->cur_un_pts[i].y - it->second.y) / dt)};
            }
            t->pts_velocity.push_back(v);
        }
    } else {
        for (size_t i = 0; i < t->cur_pts.size(); i++) t->pts_velocity.push_back(Pt{0, 0});
    }
    t->prev_un_pts_map = t->cur_un_pts_map;
}

// ---- one image step of a batch ------------------------------------------------------------------
struct ImageMsg {
    int active;
    const uint8_t* img;
    double stamp;
    int pub;
};

// Phase A: readImage up to the LK launch (feature_tracker.cpp:81-113): descriptor, points, frame staging.
void step_prepare(vt_tracker* t, const ImageMsg& m, size_t stride, bool on_device) {
    vt_batch* b = t->batch;
    vb::FeSeq& q = b->h_seq[t->member];
    const int rows = t->cfg.rows, cols = t->cfg.cols;
    t->status = VT_OK;
    t->step_active = true;
    t->step_pub = m.pub != 0;
    t->step_detect = false;
    t->cur_time = m.stamp;
    t->h2d_bytes = on_device ? 0 : (size_t)rows * cols;
    t->d2h_bytes = 0;
    t->step_first = !t->have_img;
    t->have_img = true;
    q.track = 1;
    q.detect = 0;
    q.equalize = t->cfg.equalize ? 1 : 0;
    if (on_device) {
        q.raw = m.img;
        q.raw_pitch = (int)stride;
    } else {
        for (int y = 0; y < rows; y++) std::memcpy(t->h_img + (size_t)y * cols, m.img + (size_t)y * stride, cols);
        q.raw = t->d_raw;
        q.raw_pitch = b->raw_pitch;
    }
    q.lut = t->d_lut;
    // prev = cur = forw = img on the very first frame: the pyramid built now is also the current one
    q.forw = t->pyr[t->cur ^ 1].view;
    q.cur = t->step_first ? q.forw : t->pyr[t->cur].view;
    t->forw_pts.clear();
    const int n = t->step_first ? 0 : (int)t->cur_pts.size();
    t->step_n = n;
    if (n) std::memcpy(t->h.pts_in, t->cur_pts.data(), (size_t)n * sizeof(Pt));
    q.n_pts = n;
    q.pts_in = t->d.pts_in;
    q.pts_out = t->d.pts_out;
    q.status = t->d.status;
    t->h2d_bytes += (size_t)n * sizeof(Pt) + sizeof(vb::FeSeq);
    t->d2h_bytes += (size_t)n * (sizeof(Pt) + 1);
}

// Phase B: the culls after LK, and on publishing frames rejectWithF + setMask (feature_tracker.cpp:115-146).
void step_after_track(vt_tracker* t) {
    vt_batch* b = t->batch;
    vb::FeSeq& q = b->h_seq[t->member];
    q.track = 0;
    const int n = t->step_n;
    if (n) {
        t->forw_pts.assign(reinterpret_cast<Pt*>(t->h.pts_out), reinterpret_cast<Pt*>(t->h.pts_out) + n);
        // status already includes the inBorder() cull (fused into the LK kernel)
        compact(t->cur_pts, t->h.status);
        compact(t->forw_pts, t->h.status);
        compact(t->ids, t->h.status);
        compact(t->cur_un_pts, t->h.status);
        compact(t->track_cnt, t->h.status);
    }
    for (auto& c : t->track_cnt) c++;
    t->n_pts.clear();
    if (!t->step_pub) return;
    reject_with_f(t);
    const int kept = set_mask(t);
    const int n_max_cnt = t->cfg.max_cnt - (int)t->forw_pts.size();
    if (n_max_cnt <= 0) return;
    t->step_detect = true;
    t->step_kept = kept;
    t->step_max_new = n_max_cnt;
    q.detect = 1;
    q.use_mask = 1;
    q.det_img = q.forw.img[0];
    q.det_pitch = q.forw.pitch[0];
    q.n_centres = kept;
    q.mask = t->d_mask;
    q.mask_init = t->cfg.fisheye ? t->d_fisheye.get() : nullptr;
    q.centres = t->d.centres;
    q.eig = t->d_eig;
    q.keys = t->d_keys;
    q.count = t->d.counts;
    q.maxv = reinterpret_cast<unsigned*>(t->d.counts + vb::FE_COUNT_MAXV);
    q.cell_cnt = t->d_cell_cnt;
    q.cell_pts = t->d_cell_pts;
    q.new_pts = t->d.new_pts;
    q.max_corners = n_max_cnt;
    t->h2d_bytes += (size_t)kept * 2 * sizeof(int) + sizeof(vb::FeSeq);
    t->d2h_bytes += 4 * sizeof(int) + (size_t)n_max_cnt * 2 * sizeof(float);
}

// Phase C: addPoints, rotation of the image / point sets, undistortedPoints, updateID (feature_tracker.cpp:148-167,
// feature_tracker_node.cpp:103-111).
void step_finish(vt_tracker* t) {
    if (t->step_detect) {
        if (t->h.counts[vb::FE_COUNT_CANDIDATES] > t->key_capacity) {
            t->err = "Shi-Tomasi candidate buffer overflow";
            t->status = VT_ERR_CAPACITY;
        } else {
            const int n_new = t->h.counts[vb::FE_COUNT_SELECTED];
            for (int i = 0; i < n_new; i++) t->n_pts.push_back(Pt{t->h.new_pts[2 * i], t->h.new_pts[2 * i + 1]});
        }
    }
    if (t->step_pub)
        for (auto& p : t->n_pts) {  // addPoints (feature_tracker.cpp:71-79)
            t->forw_pts.push_back(p);
            t->ids.push_back(-1);
            t->track_cnt.push_back(1);
        }
    t->cur ^= 1;  // cur_img = forw_img (prev_img is never read again by the hot path)
    t->cur_pts = t->forw_pts;
    undistorted_points(t);
    t->prev_time = t->cur_time;
    for (size_t i = 0; i < t->ids.size(); i++)  // updateID loop of img_callback (feature_tracker_node.cpp:103-111)
        if (t->ids[i] == -1) t->ids[i] = t->n_id++;
    t->step_active = false;
}

vb::FeShape base_shape(const vt_batch* b) {
    vb::FeShape sh{};
    sh.S = b->S;
    sh.rows = b->cfg.rows;
    sh.cols = b->cfg.cols;
    sh.nlev = b->nlev;
    sh.min_dist = b->cfg.min_dist;
    sh.key_capacity = b->members[0]->key_capacity;
    return sh;
}

// readImage for every member with msgs[k].active: all of them advance by one image together.
int batch_read_image(vt_batch* b, const ImageMsg* msgs, size_t stride, bool on_device) {
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaSetDevice(b->cfg.device));
    const int S = b->S;
    static const bool trace = std::getenv("VINSB200_TRACE") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b2) { return std::chrono::duration<double, std::milli>(b2 - a).count(); };
    const auto t0 = now();
    b->last_launches = 0;
    b->pool->run(S, [&](int k) {
        vt_tracker* t = b->members[k].get();
        vb::FeSeq& q = b->h_seq[k];
        q.track = q.detect = 0;
        q.n_pts = 0;
        t->step_active = false;
        t->status = VT_OK;
        if (msgs[k].active) step_prepare(t, msgs[k], stride, on_device);
    });
    vb::FeShape sh = base_shape(b);
    int first_active = -1, last_active = -1;
    for (int k = 0; k < S; k++) {
        const vb::FeSeq& q = b->h_seq[k];
        if (!q.track) continue;
        if (first_active < 0) first_active = k;
        last_active = k;
        sh.any_track = 1;
        sh.any_equalize |= q.equalize;
        sh.max_pts = std::max(sh.max_pts, q.n_pts);
    }
    if (!sh.any_track) return VT_OK;
    const auto t1 = now();
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaEventRecord(b->ev0, b->stream));
    if (!on_device) {  // the frames of members first_active..last_active travel in one copy
        const int rows = b->cfg.rows, cols = b->cfg.cols;
        VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpy2DAsync(b->d_raw + (size_t)first_active * rows * b->raw_pitch, b->raw_pitch,
                                   b->h_img + (size_t)first_active * rows * cols, cols, cols, (size_t)rows * (last_active - first_active + 1),
                                   cudaMemcpyHostToDevice, b->stream));
    }
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpyAsync(b->d_seq, b->h_seq, sizeof(vb::FeSeq) * S, cudaMemcpyHostToDevice, b->stream));
    if (sh.max_pts > 0) VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpyAsync(b->d_up, b->h_up, b->ar.centres, cudaMemcpyHostToDevice, b->stream));
    vb::launch_track(b->d_seq, sh, b->stream, &b->last_launches, &b->prof);
    if (sh.max_pts > 0) VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpyAsync(b->h_dn, b->d_dn, b->ar.track_bytes, cudaMemcpyDeviceToHost, b->stream));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaStreamSynchronize(b->stream));
    const auto t2 = now();
    b->pool->run(S, [&](int k) {
        if (b->members[k]->step_active) step_after_track(b->members[k].get());
    });
    const auto t3 = now();
    for (int k = 0; k < S; k++) {
        const vb::FeSeq& q = b->h_seq[k];
        if (!q.detect) continue;
        sh.any_detect = 1;
        sh.max_centres = std::max(sh.max_centres, q.n_centres);
    }
    if (sh.any_detect) {
        VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpyAsync(b->d_seq, b->h_seq, sizeof(vb::FeSeq) * S, cudaMemcpyHostToDevice, b->stream));
        if (sh.max_centres > 0)
            VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpyAsync(b->d_up + b->ar.centres, b->h_up + b->ar.centres, b->ar.up_bytes - b->ar.centres,
                                     cudaMemcpyHostToDevice, b->stream));
        vb::launch_detect(b->d_seq, sh, b->d_halfw, b->stream, &b->last_launches, &b->prof);
        VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpyAsync(b->h_dn + b->ar.counts, b->d_dn + b->ar.counts, b->ar.dn_bytes - b->ar.counts,
                                 cudaMemcpyDeviceToHost, b->stream));
    }
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaEventRecord(b->ev1, b->stream));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaEventSynchronize(b->ev1));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaGetLastError());
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaEventElapsedTime(&b->last_ms, b->ev0, b->ev1));
    const auto t4 = now();
    b->pool->run(S, [&](int k) {
        if (b->members[k]->step_active) step_finish(b->members[k].get());
    });
    if (trace)
        std::fprintf(stderr, "[vt_batch] prepare %.3f track(gpu) %.3f host %.3f detect(gpu) %.3f finish %.3f ms (S=%d detect=%d)\n", ms(t0, t1), ms(t1, t2),
                     ms(t2, t3), ms(t3, t4), ms(t4, now()), S, sh.any_detect);
    return vb::roll_up(b, VT_OK);
}

// img_callback's gating (feature_tracker_node.cpp:28-62): returns -1 when readImage is due (pub decided), else the
// node result (0) with *restart set when the discontinuity rule fired.
int node_gate(vt_tracker* t, double stamp, int* restart, bool* pub) {
    if (restart) *restart = 0;
    if (t->first_image_flag) {
        t->first_image_flag = false;
        t->first_image_time = stamp;
        t->last_image_time = stamp;
        return 0;
    }
    if (stamp - t->last_image_time > 1.0 || stamp < t->last_image_time) {
        t->first_image_flag = true;
        t->last_image_time = 0;
        t->pub_count = 1;
        if (restart) *restart = 1;
        return 0;
    }
    t->last_image_time = stamp;
    if (std::round(1.0 * t->pub_count / (stamp - t->first_image_time)) <= t->cfg.freq) {
        *pub = true;
        if (std::abs(1.0 * t->pub_count / (stamp - t->first_image_time) - t->cfg.freq) < 0.01 * t->cfg.freq) {
            t->first_image_time = stamp;
            t->pub_count = 0;
        }
    } else
        *pub = false;
    return -1;
}

int node_after(vt_tracker* t, bool pub) {
    if (pub) {
        t->pub_count++;
        if (!t->init_pub) {
            t->init_pub = true;
            return 1;
        }
        return 2;
    }
    return 1;
}

// Creates member k and appends it to the batch.
int create_member(vt_batch* b, int k) {
    std::unique_ptr<vt_tracker> t(new vt_tracker());
    t->cfg = b->cfg;
    t->cfg.fisheye_mask = nullptr;
    t->batch = b;
    t->member = k;
    const vt_config* cfg = &b->cfg;
    const int rows = cfg->rows, cols = cfg->cols;
    const size_t npx = (size_t)rows * cols;
    t->capacity = b->capacity;
    if (cfg->fisheye) {  // own a copy first: setMask reads it on the host
        t->owned_fisheye_mask.assign(cfg->fisheye_mask, cfg->fisheye_mask + npx);
        t->cfg.fisheye_mask = t->owned_fisheye_mask.data();
    }
    VB_CUDA_CHECK(b, VT_ERR_CUDA, t->d_lut.alloc(64 * 256));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, alloc_pyramid(t.get(), t->pyr[0]));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, alloc_pyramid(t.get(), t->pyr[1]));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, t->d_mask.alloc(npx));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, t->d_eig.alloc(npx));
    t->key_capacity = 1;
    while ((size_t)t->key_capacity < npx / 8) t->key_capacity <<= 1;  // local maxima of a 3x3 NMS: < npx/4 in practice
    VB_CUDA_CHECK(b, VT_ERR_CUDA, t->d_keys.alloc((size_t)t->key_capacity));
    const int cell = cfg->min_dist, gw = (cols + cell - 1) / cell, gh = (rows + cell - 1) / cell;
    VB_CUDA_CHECK(b, VT_ERR_CUDA, t->d_cell_cnt.alloc((size_t)gw * gh));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, t->d_cell_pts.alloc((size_t)gw * gh * 8));
    if (cfg->fisheye) {
        VB_CUDA_CHECK(b, VT_ERR_CUDA, t->d_fisheye.alloc(npx));
        VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpy(t->d_fisheye, t->owned_fisheye_mask.data(), npx, cudaMemcpyHostToDevice));
    }
    t->halfw = disc_half_widths(cfg->min_dist);
    t->d_raw = b->d_raw + (size_t)k * rows * b->raw_pitch;
    t->h_img = b->h_img + (size_t)k * npx;
    t->h = arena_slots(b->ar, b->h_up, b->h_dn, k);
    t->d = arena_slots(b->ar, b->d_up, b->d_dn, k);
    t->cfg.freq = b->cfg.freq;
    t->cfg.focal_length = b->cfg.focal_length;
    b->members.push_back(std::move(t));
    return VT_OK;
}

}  // namespace

extern "C" {

int vt_batch_create(const vt_config* cfg, int n, vt_batch** out) {
    if (!cfg || !out || n < 1 || n > 4096) return VT_ERR_INVALID;
    *out = nullptr;
    if (cfg->rows < 32 || cfg->cols < 32 || cfg->max_cnt <= 0 || cfg->min_dist < 1 ||
        cfg->camera_model < VT_CAMERA_PINHOLE || cfg->camera_model > VT_CAMERA_KANNALA_BRANDT || (cfg->fisheye && !cfg->fisheye_mask))
        return VT_ERR_INVALID;
    if (!vb::device_available(cfg->device)) return VT_ERR_NO_DEVICE;
    std::unique_ptr<vt_batch, void (*)(vt_batch*)> b(new vt_batch(), vt_batch_destroy);
    b->cfg = *cfg;
    if (b->cfg.freq == 0) b->cfg.freq = 100;
    if (b->cfg.focal_length == 0) b->cfg.focal_length = 460;
    b->S = n;
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaSetDevice(cfg->device));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->stream.create());
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->ev0.create());
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->ev1.create());
    const int rows = cfg->rows, cols = cfg->cols;
    const size_t npx = (size_t)rows * cols, S = (size_t)n;
    b->raw_pitch = align_up(cols, 64);
    b->capacity = std::max(cfg->max_cnt, 16);
    b->nlev = lk_levels(rows, cols, 21, 3);
    b->ar = arena_layout(S, (size_t)b->capacity);
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->d_raw.alloc(S * rows * b->raw_pitch));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->h_img.alloc(S * npx));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->d_up.alloc(b->ar.up_bytes));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->h_up.alloc(b->ar.up_bytes));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->d_dn.alloc(b->ar.dn_bytes));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->h_dn.alloc(b->ar.dn_bytes));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->d_seq.alloc(S));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->h_seq.alloc(S));
    std::memset(b->h_seq, 0, sizeof(vb::FeSeq) * S);
    const std::vector<int> hw = disc_half_widths(cfg->min_dist);
    VB_CUDA_CHECK(b, VT_ERR_CUDA, b->d_halfw.alloc(hw.size()));
    VB_CUDA_CHECK(b, VT_ERR_CUDA, cudaMemcpy(b->d_halfw, hw.data(), hw.size() * sizeof(int), cudaMemcpyHostToDevice));
    for (int k = 0; k < n; k++) {
        const int rc = create_member(b.get(), k);
        if (rc) return rc;
    }
    b->pool.reset(new vb::HostPool(vb::HostPool::default_workers(n)));
    *out = b.release();
    return VT_OK;
}

void vt_batch_destroy(vt_batch* b) {
    vb::destroy_batch(b, [b] {
        if (b->stream) cudaStreamSynchronize(b->stream);
        b->pool.reset();
    });
}

int vt_batch_size(const vt_batch* b) { return vb::batch_size(b, VT_ERR_INVALID); }
vt_tracker* vt_batch_member(vt_batch* b, int k) { return vb::batch_member(b, k); }
const char* vt_batch_last_error(const vt_batch* b) { return vb::batch_last_error(b); }

int vt_batch_read_image(vt_batch* b, const int* active, const uint8_t* const* imgs, size_t row_stride, const double* cur_times,
                        const int* pub_this_frame, int images_on_device) {
    if (!b || !imgs || !cur_times || !pub_this_frame || row_stride < (size_t)b->cfg.cols) return VT_ERR_INVALID;
    std::vector<ImageMsg> msgs(b->S);
    for (int k = 0; k < b->S; k++) {
        msgs[k] = ImageMsg{active ? (active[k] != 0) : 1, imgs[k], cur_times[k], pub_this_frame[k]};
        if (msgs[k].active && !imgs[k]) return VT_ERR_INVALID;
    }
    return batch_read_image(b, msgs.data(), row_stride, images_on_device != 0);
}

int vt_batch_node_image(vt_batch* b, const int* active, const uint8_t* const* imgs, size_t row_stride, const double* stamps,
                        int images_on_device, int* results, int* restarts) {
    if (!b || !imgs || !stamps || !results || row_stride < (size_t)b->cfg.cols) return VT_ERR_INVALID;
    std::vector<ImageMsg> msgs(b->S);
    for (int k = 0; k < b->S; k++) {
        msgs[k] = ImageMsg{0, imgs[k], stamps[k], 0};
        results[k] = 0;
        if (restarts) restarts[k] = 0;
        if (active && !active[k]) continue;
        if (!imgs[k]) return VT_ERR_INVALID;
        bool pub = false;
        const int r = node_gate(b->members[k].get(), stamps[k], restarts ? restarts + k : nullptr, &pub);
        if (r >= 0) continue;  // first frame or restart: the image is consumed without tracking
        msgs[k].active = 1;
        msgs[k].pub = pub ? 1 : 0;
    }
    const int rc = batch_read_image(b, msgs.data(), row_stride, images_on_device != 0);
    if (rc) return rc;
    for (int k = 0; k < b->S; k++)
        if (msgs[k].active) results[k] = node_after(b->members[k].get(), msgs[k].pub != 0);
    return VT_OK;
}

int vt_batch_last_timing(const vt_batch* b, float* device_ms, int* kernel_launches) {
    if (!b) return VT_ERR_INVALID;
    if (device_ms) *device_ms = b->last_ms;
    if (kernel_launches) *kernel_launches = b->last_launches;
    return VT_OK;
}

int vt_batch_set_profile(vt_batch* b, int on) { return vb::set_profile(b, on, VT_ERR_INVALID, VT_ERR_CUDA); }

int vt_batch_kernel_times(const vt_batch* b, double* ms6, int* count6) { return vb::kernel_times(b, ms6, count6, 6, VT_ERR_INVALID); }

int vt_create(const vt_config* cfg, vt_tracker** out) { return vb::create_standalone(vt_batch_create, cfg, out, VT_ERR_INVALID); }

void vt_destroy(vt_tracker* t) { vb::destroy_standalone(t, vt_batch_destroy); }

const char* vt_last_error(const vt_tracker* t) { return vb::last_error(t); }

static int read_image_single(vt_tracker* t, const uint8_t* img, size_t stride, double cur_time, int pub, bool on_device) {
    if (!t || !img || stride < (size_t)t->cfg.cols) return VT_ERR_INVALID;
    if (const int rc = vb::refuse_member(t, VT_ERR_INVALID, "per-handle image call on a member of a batch: use vt_batch_read_image / vt_batch_node_image"))
        return rc;
    t->err.clear();
    ImageMsg m{1, img, cur_time, pub};
    return batch_read_image(t->batch, &m, stride, on_device);
}

int vt_read_image(vt_tracker* t, const uint8_t* img, size_t row_stride, double cur_time, int pub_this_frame) {
    return read_image_single(t, img, row_stride, cur_time, pub_this_frame, false);
}

int vt_read_image_device(vt_tracker* t, const uint8_t* d_img, size_t row_stride, double cur_time, int pub_this_frame) {
    return read_image_single(t, d_img, row_stride, cur_time, pub_this_frame, true);
}

int vt_count(const vt_tracker* t) { return t ? (int)t->cur_pts.size() : VT_ERR_INVALID; }

int vt_get(const vt_tracker* t, int* ids, int* track_cnt, float* cur_pts, float* cur_un_pts, float* pts_velocity) {
    if (!t) return VT_ERR_INVALID;
    const size_t n = t->cur_pts.size();
    if (ids) std::memcpy(ids, t->ids.data(), n * sizeof(int));
    if (track_cnt) std::memcpy(track_cnt, t->track_cnt.data(), n * sizeof(int));
    if (cur_pts) std::memcpy(cur_pts, t->cur_pts.data(), n * sizeof(Pt));
    if (cur_un_pts) std::memcpy(cur_un_pts, t->cur_un_pts.data(), n * sizeof(Pt));
    if (pts_velocity) std::memcpy(pts_velocity, t->pts_velocity.data(), n * sizeof(Pt));
    return (int)n;
}

static int node_image_single(vt_tracker* t, const uint8_t* img, size_t row_stride, double stamp, int* restart, bool on_device) {
    if (!t) return VT_ERR_INVALID;
    bool pub = false;
    const int r = node_gate(t, stamp, restart, &pub);
    if (r >= 0) return r;
    const int rc = read_image_single(t, img, row_stride, stamp, pub, on_device);
    if (rc) return rc;
    return node_after(t, pub);
}

int vt_node_image(vt_tracker* t, const uint8_t* img, size_t row_stride, double stamp, int* restart) {
    return node_image_single(t, img, row_stride, stamp, restart, false);
}

int vt_node_image_device(vt_tracker* t, const uint8_t* d_img, size_t row_stride, double stamp, int* restart) {
    return node_image_single(t, d_img, row_stride, stamp, restart, true);
}

int vt_node_pack(const vt_tracker* t, int capacity, float* xy_un, float* id_of_point, float* u_of_point,
                 float* v_of_point, float* velocity_x, float* velocity_y) {
    if (!t) return VT_ERR_INVALID;
    int k = 0;
    for (size_t j = 0; j < t->ids.size(); j++) {
        if (t->track_cnt[j] <= 1) continue;
        if (k >= capacity) return VT_ERR_CAPACITY;
        xy_un[2 * k] = t->cur_un_pts[j].x;
        xy_un[2 * k + 1] = t->cur_un_pts[j].y;
        id_of_point[k] = (float)(t->ids[j] * 1 + 0);
        u_of_point[k] = t->cur_pts[j].x;
        v_of_point[k] = t->cur_pts[j].y;
        velocity_x[k] = t->pts_velocity[j].x;
        velocity_y[k] = t->pts_velocity[j].y;
        k++;
    }
    return k;
}

int vt_debug_fundamental_ransac(const float* pts1, const float* pts2, int n, double threshold, double confidence, uint8_t* status) {
    if (!pts1 || !pts2 || !status || n < 0) return VT_ERR_INVALID;
    return vb::fundamental_ransac_mask(pts1, pts2, n, threshold, confidence, status) ? 1 : 0;
}

int vt_debug_fundamental_ransac_model(const float* pts1, const float* pts2, int n, double threshold, double confidence, uint8_t* status, double* F9) {
    if (!pts1 || !pts2 || !status || !F9 || n < 0) return VT_ERR_INVALID;
    return vb::fundamental_ransac(pts1, pts2, n, threshold, confidence, status, F9) ? 1 : 0;
}

int vt_debug_lift_projective(const double* intrinsics8, const double* px, int n, double* out_xy) {
    if (!intrinsics8 || !px || !out_xy || n < 0) return VT_ERR_INVALID;
    vt_config c{};
    for (int i = 0; i < 8; i++) c.intrinsics[i] = intrinsics8[i];
    for (int k = 0; k < n; k++) lift_projective(c, px[2 * k], px[2 * k + 1], out_xy[2 * k], out_xy[2 * k + 1]);
    return VT_OK;
}

int vt_debug_lift_projective_model(int camera_model, const double* intrinsics8, double xi, const double* px, int n, double* out_xy) {
    if (!intrinsics8 || !px || !out_xy || n < 0 || camera_model < VT_CAMERA_PINHOLE || camera_model > VT_CAMERA_KANNALA_BRANDT)
        return VT_ERR_INVALID;
    vt_config c{};
    c.camera_model = camera_model;
    c.xi = xi;
    for (int i = 0; i < 8; i++) c.intrinsics[i] = intrinsics8[i];
    for (int k = 0; k < n; k++) lift_projective(c, px[2 * k], px[2 * k + 1], out_xy[2 * k], out_xy[2 * k + 1]);
    return VT_OK;
}

int vt_debug_disc_half_widths(int radius, int* out) {
    if (radius < 0 || !out) return VT_ERR_INVALID;
    const std::vector<int> hw = disc_half_widths(radius);
    for (int d = 0; d <= radius; d++) out[d] = hw[d];
    return VT_OK;
}

int vt_last_timing(const vt_tracker* t, float* device_ms, int* kernel_launches) {
    return t ? vt_batch_last_timing(t->batch, device_ms, kernel_launches) : VT_ERR_INVALID;
}

int vt_set_profile(vt_tracker* t, int on) { return t ? vt_batch_set_profile(t->batch, on) : VT_ERR_INVALID; }

int vt_kernel_times(const vt_tracker* t, double* ms6, int* count6) { return t ? vt_batch_kernel_times(t->batch, ms6, count6) : VT_ERR_INVALID; }

int vt_last_traffic(const vt_tracker* t, double* h2d_bytes, double* d2h_bytes) {
    if (!t) return VT_ERR_INVALID;
    if (h2d_bytes) *h2d_bytes = (double)t->h2d_bytes;
    if (d2h_bytes) *d2h_bytes = (double)t->d2h_bytes;
    return VT_OK;
}

int vt_debug_equalized(vt_tracker* t, int level, uint8_t* out, int* rows, int* cols) {
    if (!t || !t->have_img) return VT_ERR_INVALID;
    const vb::PyramidView& v = t->pyr[t->cur].view;
    if (level < 0 || level > v.nlev) return VT_ERR_INVALID;
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaSetDevice(t->cfg.device));
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpy2D(out, v.cols[level], v.img[level], v.pitch[level], v.cols[level], v.rows[level],
                         cudaMemcpyDeviceToHost));
    if (rows) *rows = v.rows[level];
    if (cols) *cols = v.cols[level];
    return VT_OK;
}

int vt_debug_gftt(vt_tracker* t, const uint8_t* img, size_t row_stride, const uint8_t* mask, int max_corners,
                  float* corners, int* n_candidates, float* eig_out) {
    if (!t || !img || max_corners <= 0 || max_corners > t->capacity) return VT_ERR_INVALID;
    vt_batch* b = t->batch;
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaSetDevice(t->cfg.device));
    const int rows = t->cfg.rows, cols = t->cfg.cols;
    vb::DeviceArray<uint8_t> d_user_mask;
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpy2DAsync(t->d_raw, b->raw_pitch, img, row_stride, cols, rows, cudaMemcpyHostToDevice, b->stream));
    if (mask) {
        VB_CUDA_CHECK(t, VT_ERR_CUDA, d_user_mask.alloc((size_t)rows * cols));
        VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpyAsync(d_user_mask, mask, (size_t)rows * cols, cudaMemcpyHostToDevice, b->stream));
    }
    vb::FeSeq& q = b->h_seq[t->member];
    std::memset(&q, 0, sizeof(q));
    q.detect = 1;
    q.use_mask = mask ? 1 : 0;
    q.det_img = t->d_raw;
    q.det_pitch = b->raw_pitch;
    q.mask = t->d_mask;
    q.mask_init = d_user_mask;
    q.eig = t->d_eig;
    q.keys = t->d_keys;
    q.count = t->d.counts;
    q.maxv = reinterpret_cast<unsigned*>(t->d.counts + vb::FE_COUNT_MAXV);
    q.cell_cnt = t->d_cell_cnt;
    q.cell_pts = t->d_cell_pts;
    q.new_pts = t->d.new_pts;
    q.max_corners = max_corners;
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpyAsync(b->d_seq, b->h_seq, sizeof(vb::FeSeq) * b->S, cudaMemcpyHostToDevice, b->stream));
    vb::FeShape sh = base_shape(b);
    sh.any_detect = 1;
    vb::launch_detect(b->d_seq, sh, b->d_halfw, b->stream, nullptr, nullptr);
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpyAsync(b->h_dn + b->ar.counts, b->d_dn + b->ar.counts, b->ar.dn_bytes - b->ar.counts,
                            cudaMemcpyDeviceToHost, b->stream));
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaStreamSynchronize(b->stream));
    q.detect = 0;
    if (t->h.counts[vb::FE_COUNT_CANDIDATES] > t->key_capacity) {
        t->err = "Shi-Tomasi candidate buffer overflow";
        return VT_ERR_CAPACITY;
    }
    const int n = t->h.counts[vb::FE_COUNT_SELECTED];
    if (n_candidates) *n_candidates = t->h.counts[vb::FE_COUNT_CANDIDATES];
    std::memcpy(corners, t->h.new_pts, (size_t)n * 2 * sizeof(float));
    if (eig_out) VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpy(eig_out, t->d_eig, (size_t)rows * cols * sizeof(float), cudaMemcpyDeviceToHost));
    return n;
}

int vt_debug_lk(vt_tracker* t, const uint8_t* prev, const uint8_t* next, size_t row_stride, const float* pts, int n,
                float* next_pts, uint8_t* status) {
    if (!t || !prev || !next || n < 0 || n > t->capacity) return VT_ERR_INVALID;
    vt_batch* b = t->batch;
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaSetDevice(t->cfg.device));
    const int rows = t->cfg.rows, cols = t->cfg.cols;
    for (int k = 0; k < 2; k++) {
        DevicePyramid& p = t->pyr[k];
        VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpy2DAsync(const_cast<uint8_t*>(p.view.img[0]), p.view.pitch[0], k == 0 ? prev : next, row_stride,
                                  cols, rows, cudaMemcpyHostToDevice, b->stream));
    }
    vb::FeSeq& q = b->h_seq[t->member];
    std::memset(&q, 0, sizeof(q));
    q.track = 1;
    q.cur = t->pyr[0].view;
    q.forw = t->pyr[1].view;
    q.n_pts = n;
    q.pts_in = t->d.pts_in;
    q.pts_out = t->d.pts_out;
    q.status = t->d.status;
    if (n) std::memcpy(t->h.pts_in, pts, (size_t)n * 2 * sizeof(float));
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpyAsync(b->d_seq, b->h_seq, sizeof(vb::FeSeq) * b->S, cudaMemcpyHostToDevice, b->stream));
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpyAsync(b->d_up, b->h_up, b->ar.centres, cudaMemcpyHostToDevice, b->stream));
    vb::FeShape sh = base_shape(b);
    sh.any_track = 1;
    sh.max_pts = n;
    vb::launch_pyramid_only(b->d_seq, sh, 1, b->stream);
    vb::launch_pyramid_only(b->d_seq, sh, 0, b->stream);
    vb::launch_lk_only(b->d_seq, sh, b->stream);
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaMemcpyAsync(b->h_dn, b->d_dn, b->ar.track_bytes, cudaMemcpyDeviceToHost, b->stream));
    VB_CUDA_CHECK(t, VT_ERR_CUDA, cudaStreamSynchronize(b->stream));
    q.track = 0;
    if (n) {
        std::memcpy(next_pts, t->h.pts_out, (size_t)n * 2 * sizeof(float));
        std::memcpy(status, t->h.status, n);
    }
    t->have_img = false;  // the pyramids no longer belong to the tracking state
    return VT_OK;
}

}  // extern "C"
