// ve_* C ABI: host shim of the reference's Estimator / FeatureManager (vins_estimator/src/estimator.cpp,
// feature_manager.cpp) around the CUDA BA path.  Bookkeeping that the reference does on the host stays on the
// host (window arrays, feature tracks, slide/re-anchor logic); IMU pre-integration, factor linearisation, the
// trust-region solve, the gauge re-anchoring of double2vector and the marginalisation run on the GPU with all problem
// data resident in HBM.
//
// Execution model: estimators are members of a batch (ve_batch; a stand-alone handle is a batch of one).  A frame of
// the batch is   prepare (host, per member, parallel)  ->  ONE host-to-device copy of the packed inputs  ->  one launch
// chain for all members (pre-integration jobs, 8-iteration solve, re-anchoring, marginalisation)  ->  ONE device-to-host
// copy of the results  ->  finish (host, per member, parallel).  The host waits once per frame (for the results); the
// marginalisation keeps running behind that point and is only awaited by the next frame's kernels on the same stream.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "ba_kernels.h"
#include "ba_layout.h"
#include "batch_host.h"
#include "cuda_check.h"
#include "hostpool.h"
#include "initial.h"
#include "rotation.h"
#include "vinsb200/estimator.h"

using vb::Mat3;
using vb::Quat;
using vb::Vec3;

namespace {

struct FeaturePerFrame {  // feature_manager.h:19-46
    Vec3 point;
    double u, v, vx, vy, cur_td;
};
struct FeaturePerId {  // feature_manager.h:48-72
    int feature_id, start_frame;
    std::vector<FeaturePerFrame> feature_per_frame;
    int used_num = 0;
    double estimated_depth = -1.0;
    int solve_flag = 0;
    int endFrame() const { return start_frame + (int)feature_per_frame.size() - 1; }
};

struct SeedRow {
    double t;
    Vec3 P, V;
    Mat3 R;
};

struct PriorBlock {
    int type, index, off, size;  // type 0 pose, 1 speed-bias, 2 ex pose, 3 td; size = local size
};

enum FrameStage { STAGE_DONE = 0, STAGE_INIT_SOLVE = 1, STAGE_RUN_SOLVE = 2 };

}  // namespace

struct ve_estimator : vb::MemberBase<ve_batch> {
    ve_config cfg{};
    int W = 10;
    // ---- Estimator state (estimator.h:65-115)
    int solver_flag = 0;           // INITIAL = 0, NON_LINEAR = 1
    int marginalization_flag = 0;  // MARGIN_OLD = 0, MARGIN_SECOND_NEW = 1
    Vec3 g;
    Mat3 ric;
    Vec3 tic;
    std::vector<Vec3> Ps, Vs, Bas, Bgs;
    std::vector<Mat3> Rs;
    double td = 0;
    Mat3 back_R0, last_R, last_R0;
    Vec3 back_P0, last_P, last_P0;
    std::vector<double> Headers;
    Vec3 acc_0, gyr_0;
    std::vector<std::vector<double>> dt_buf;
    std::vector<std::vector<Vec3>> acc_buf, gyr_buf;
    int frame_count = 0;
    bool first_imu = false, failure_occur = false;
    std::vector<FeaturePerId> feature;  // FeatureManager::feature (std::list in the reference; order preserved)
    int last_track_num = 0;
    std::vector<SeedRow> seeds;
    Vec3 seed_ba, seed_bg;
    // relocalisation (estimator.h:125-138): set by ve_set_relo_frame, consumed by the next solve
    bool relocalization_info = false, fr_relo = false;
    double relo_frame_stamp = 0;
    int relo_frame_index = 0, relo_frame_local_index = 0;
    std::vector<double> match_points;  // x, y, feature id per match, ascending id
    double relo_Pose[7] = {0, 0, 0, 0, 0, 0, 1};
    std::vector<std::array<double, 7>> para_Pose;  // the window poses as last packed by vector2double (post-solve, pre-slide)
    Mat3 drift_correct_r, prev_relo_r;
    Vec3 drift_correct_t, prev_relo_t, relo_relative_t;
    Quat relo_relative_q;
    double relo_relative_yaw = 0;
    int n_relo_factors = 0, n_relo_solves = 0;
    // ESTIMATE_EXTRINSIC == 2 (estimator.cpp:140-156): the camera-IMU rotation is calibrated online before the initialisation
    vb::init::ExRotation initial_ex_rotation;
    bool ex_calib_pending = false;  // ESTIMATE_EXTRINSIC is still 2
    Mat3 RIC;                       // RIC[0]: the configured rotation, replaced by the calibrated one
    // initialisation bookkeeping while solver_flag == INITIAL (estimator.h:117-119: all_image_frame, tmp_pre_integration)
    std::vector<vb::init::ImageFrame> all_image_frame;  // ascending stamps (std::map<double, ImageFrame> in the reference)
    vb::init::Preint tmp_pre;
    double initial_timestamp = 0;
    bool self_initialised = false;
    int init_failures = 0, init_l = -1, init_iterations = 0;
    double init_scale = 0, init_cost = 0;
    // pre-integration slots: frame -> slot, per-slot host mirror of what the device slot was created with
    std::vector<int> slot_of;
    std::vector<bool> slot_valid;
    std::vector<size_t> flushed;    // samples of dt_buf[frame] already handed to the device
    std::vector<double> sum_dt;     // per frame
    std::vector<Vec3> lin_acc, lin_gyr;  // linearized_acc / linearized_gyr per frame
    std::vector<bool> sqrt_dirty;   // per slot
    // device work queued since the last launch (executed in order at the head of the next frame's kernel chain)
    std::vector<vb::PreintJob> jobs;
    std::vector<double> job_samples;  // 7 doubles per record
    // prior (MarginalizationInfo) bookkeeping
    bool has_prior = false;
    int prior_n = 0, prior_buf = 0;
    std::vector<PriorBlock> prior_blocks;
    // summary
    int n_solves = 0, n_reboots = 0, last_landmarks = 0, last_visual = 0;
    vb::SolverState last_state{};
    size_t h2d_bytes = 0, d2h_bytes = 0;  // of the last process_image
    // ---- per-frame plan (prepare -> launch -> finish)
    int stage = STAGE_DONE;
    int status = VE_OK;      // of the current frame
    bool fr_marg = false;
    int fr_L = 0;
    size_t out_off = 0;      // doubles, into the batch output arena
    const double* marg_Araw = nullptr;  // device: Schur complement of the last marginalisation before the eps floor
    const double* marg_graw = nullptr;
    int marg_n = 0;
    // ---- persistent device memory of this member
    int Lmax = 0, Mmax = 0, D = 0, nmax = 0;
    vb::DeviceArray<vb::PreInt> d_preint;
    vb::DeviceArray<double> d_states1;     // x[1] (x[0] lives in the frame's input block)
    vb::DeviceArray<double> d_acc[2];      // Hpp | gp | Hpl | Hll | gl | cost
    vb::DeviceArray<double> d_S, d_Spk, d_Hfull, d_gred, d_vec, d_work;
    vb::DeviceArray<double> d_prior[2];    // A | g0 | c0 | x0
    vb::DeviceArray<double> d_marg;        // Am | bm | Araw | graw | Wglobal
};

struct ve_batch : vb::BatchBase<ve_estimator> {
    ve_config cfg{};
    // Launch groups: the members are split into G contiguous groups, each with its own streams, events and arena slices.
    // Every group runs the same launch chain over its members; the chains of different groups overlap on the GPU (the
    // single-CTA-per-member solvers of one group leave most SMs to the wide kernels of another).
    struct Group {
        int first = 0, count = 0;
        vb::Stream stream, copy_stream;
        vb::Event ev[8];  // 0 frame start, 1 after pre-integration, 2 after the solve + re-anchoring, 3 marginalisation done,
                                 // 4 results on the host, 5 marginalisation start
        size_t in_base = 0, in_cap = 0;    // bytes, slice of the input arena
        size_t out_base = 0, out_cap = 0;  // doubles, slice of the output arena
        std::atomic<size_t> in_used{0}, out_used{0};
        bool waits_results = false, has_marg = false;
    };
    int G = 1;
    std::unique_ptr<Group[]> groups;
    int members_per_group = 1;
    vb::PinnedArray<vb::BaSeq> h_seq;  // mirror of d_seq
    vb::DeviceArray<vb::BaSeq> d_seq;
    vb::PinnedArray<unsigned char> h_in;  // packed per-member input blocks of the frame
    vb::DeviceArray<unsigned char> d_in;
    vb::PinnedArray<double> h_out;        // per-member output blocks
    vb::DeviceArray<double> d_out;
    vb::KernelProfile prof;
    std::unique_ptr<vb::HostPool> pool;
    float last_ms[4] = {0, 0, 0, 0};
    int last_launches = 0;
    bool marg_timing_valid = false;
    int w_in_global = 0;            // marg_solve keeps its reduced system in global memory (large windows)
    std::vector<int> active;        // scratch: members taking part in the current frame
};

namespace {

bool usable(const ve_estimator* e, FeaturePerId& it) {  // the filter repeated all over feature_manager.cpp
    it.used_num = (int)it.feature_per_frame.size();
    return it.used_num >= 2 && it.start_frame < e->W - 2;
}

// ---- pre-integration slots: the device work is queued and runs at the head of the next frame's kernel chain -------
void init_slot(ve_estimator* e, int frame, const Vec3& a0, const Vec3& g0, const Vec3& ba, const Vec3& bg) {
    const int slot = e->slot_of[frame];
    // a new IntegrationBase supersedes whatever was queued for the slot
    e->jobs.erase(std::remove_if(e->jobs.begin(), e->jobs.end(), [&](const vb::PreintJob& j) { return j.slot == slot; }), e->jobs.end());
    if (e->jobs.empty()) e->job_samples.clear();
    vb::PreintJob j{};
    j.type = 0;
    j.slot = slot;
    j.acc0[0] = a0.x; j.acc0[1] = a0.y; j.acc0[2] = a0.z;
    j.gyr0[0] = g0.x; j.gyr0[1] = g0.y; j.gyr0[2] = g0.z;
    j.ba[0] = ba.x; j.ba[1] = ba.y; j.ba[2] = ba.z;
    j.bg[0] = bg.x; j.bg[1] = bg.y; j.bg[2] = bg.z;
    e->jobs.push_back(j);
    e->slot_valid[frame] = true;
    e->flushed[frame] = 0;
    e->sum_dt[frame] = 0;
    e->lin_acc[frame] = a0;
    e->lin_gyr[frame] = g0;
    e->sqrt_dirty[slot] = true;
}

// Queues the not-yet-integrated samples of `frame`'s buffers for its device slot.
void flush_frame(ve_estimator* e, int frame) {
    const size_t n = e->dt_buf[frame].size();
    if (!e->slot_valid[frame] || e->flushed[frame] >= n) return;
    const size_t k0 = e->flushed[frame], cnt = n - k0;
    vb::PreintJob j{};
    j.type = 1;
    j.slot = e->slot_of[frame];
    j.n = (int)cnt;
    j.sample_off = (int)(e->job_samples.size() / 7);
    for (size_t k = 0; k < cnt; k++) {
        const Vec3 &a = e->acc_buf[frame][k0 + k], &w = e->gyr_buf[frame][k0 + k];
        const double rec[7] = {e->dt_buf[frame][k0 + k], a.x, a.y, a.z, w.x, w.y, w.z};
        e->job_samples.insert(e->job_samples.end(), rec, rec + 7);
    }
    e->jobs.push_back(j);
    e->flushed[frame] = n;
    e->sqrt_dirty[e->slot_of[frame]] = true;
}

unsigned refresh_sqrt_mask(ve_estimator* e) {
    unsigned mask = 0;
    for (int f = 1; f <= e->W; f++) {
        const int s = e->slot_of[f];
        if (e->slot_valid[f] && e->sqrt_dirty[s] && e->dt_buf[f].size() > 0) {
            mask |= 1u << s;
            e->sqrt_dirty[s] = false;
        }
    }
    return mask;
}

// ---- FeatureManager (feature_manager.cpp) ------------------------------------------------------
double compensated_parallax2(const FeaturePerId& it, int frame_count) {
    const FeaturePerFrame& fi = it.feature_per_frame[frame_count - 2 - it.start_frame];
    const FeaturePerFrame& fj = it.feature_per_frame[frame_count - 1 - it.start_frame];
    const double dep_i = fi.point.z;
    const double du = fi.point.x / dep_i - fj.point.x, dv = fi.point.y / dep_i - fj.point.y;
    return std::max(0.0, std::sqrt(std::min(du * du + dv * dv, du * du + dv * dv)));
}

bool add_feature_check_parallax(ve_estimator* e, int n, const int* order, const int* ids, const double* d7, double td) {
    double parallax_sum = 0;
    int parallax_num = 0;
    e->last_track_num = 0;
    for (int k = 0; k < n; k++) {  // ascending feature id (std::map order)
        const int i = order[k];
        const double* d = d7 + 7 * i;
        const FeaturePerFrame f{Vec3(d[0], d[1], d[2]), d[3], d[4], d[5], d[6], td};
        auto it = std::find_if(e->feature.begin(), e->feature.end(), [&](const FeaturePerId& x) { return x.feature_id == ids[i]; });
        if (it == e->feature.end()) {
            FeaturePerId nf;
            nf.feature_id = ids[i];
            nf.start_frame = e->frame_count;
            nf.feature_per_frame.push_back(f);
            e->feature.push_back(nf);
        } else {
            it->feature_per_frame.push_back(f);
            e->last_track_num++;
        }
    }
    const int fc = e->frame_count;
    if (fc < 2 || e->last_track_num < 20) return true;
    for (auto& it : e->feature)
        if (it.start_frame <= fc - 2 && it.start_frame + (int)it.feature_per_frame.size() - 1 >= fc - 1) {
            parallax_sum += compensated_parallax2(it, fc);
            parallax_num++;
        }
    if (parallax_num == 0) return true;
    return parallax_sum / parallax_num >= e->cfg.keyframe_parallax / e->cfg.focal_length;
}

void triangulate(ve_estimator* e) {
    for (auto& it : e->feature) {
        if (!usable(e, it)) continue;
        if (it.estimated_depth > 0) continue;
        const int imu_i = it.start_frame;
        int imu_j = imu_i - 1;
        double A[64 * 4];
        int row = 0;
        const Vec3 t0 = e->Ps[imu_i] + e->Rs[imu_i] * e->tic;
        const Mat3 R0 = e->Rs[imu_i] * e->ric;
        for (auto& f : it.feature_per_frame) {
            imu_j++;
            const Vec3 t1 = e->Ps[imu_j] + e->Rs[imu_j] * e->tic;
            const Mat3 R1 = e->Rs[imu_j] * e->ric;
            const Vec3 t = R0.T() * (t1 - t0);
            const Mat3 Rt = (R0.T() * R1).T();
            const Vec3 mt = (Rt * t) * -1.0;
            double P[3][4];
            for (int i = 0; i < 3; i++) {
                for (int j = 0; j < 3; j++) P[i][j] = Rt(i, j);
                P[i][3] = mt[i];
            }
            const double nn = f.point.norm();
            const Vec3 fn = f.point * (1.0 / nn);
            for (int c = 0; c < 4; c++) {
                A[4 * row + c] = fn.x * P[2][c] - fn.z * P[0][c];
                A[4 * (row + 1) + c] = fn.y * P[2][c] - fn.z * P[1][c];
            }
            row += 2;
        }
        double v[4];
        vb::null_direction4(A, row, v);
        it.estimated_depth = v[2] / v[3];
        if (it.estimated_depth < 0.1) it.estimated_depth = e->cfg.init_depth;
    }
}

void remove_back_shift_depth(ve_estimator* e, const Mat3& marg_R, const Vec3& marg_P, const Mat3& new_R, const Vec3& new_P) {
    std::vector<FeaturePerId> keep;
    keep.reserve(e->feature.size());
    for (auto& it : e->feature) {
        if (it.start_frame != 0) {
            it.start_frame--;
            keep.push_back(std::move(it));
            continue;
        }
        const Vec3 uv_i = it.feature_per_frame[0].point;
        it.feature_per_frame.erase(it.feature_per_frame.begin());
        if (it.feature_per_frame.size() < 2) continue;
        const Vec3 pts_i = uv_i * it.estimated_depth;
        const Vec3 w_pts_i = marg_R * pts_i + marg_P;
        const Vec3 pts_j = new_R.T() * (w_pts_i - new_P);
        it.estimated_depth = pts_j.z > 0 ? pts_j.z : e->cfg.init_depth;
        keep.push_back(std::move(it));
    }
    e->feature.swap(keep);
}
void remove_back(ve_estimator* e) {
    std::vector<FeaturePerId> keep;
    for (auto& it : e->feature) {
        if (it.start_frame != 0)
            it.start_frame--;
        else {
            it.feature_per_frame.erase(it.feature_per_frame.begin());
            if (it.feature_per_frame.empty()) continue;
        }
        keep.push_back(std::move(it));
    }
    e->feature.swap(keep);
}
void remove_front(ve_estimator* e, int frame_count) {
    std::vector<FeaturePerId> keep;
    for (auto& it : e->feature) {
        if (it.start_frame == frame_count)
            it.start_frame--;
        else if (it.endFrame() >= frame_count - 1) {
            const int j = e->W - 1 - it.start_frame;
            it.feature_per_frame.erase(it.feature_per_frame.begin() + j);
            if (it.feature_per_frame.empty()) continue;
        }
        keep.push_back(std::move(it));
    }
    e->feature.swap(keep);
}

// ---- Estimator ---------------------------------------------------------------------------------
void set_parameter(ve_estimator* e) {
    e->tic = Vec3(e->cfg.tic[0], e->cfg.tic[1], e->cfg.tic[2]);
    e->ric = e->RIC;
    e->td = e->cfg.td;
    e->g = Vec3(0, 0, e->cfg.g_norm);
}

void clear_state(ve_estimator* e) {
    // Device-side leftovers need no wait: the slots are re-created by queued jobs, the prior is dropped (has_prior), and
    // anything still running on the batch stream is ordered before the next frame's kernels.
    e->jobs.clear();
    e->job_samples.clear();
    for (int i = 0; i <= e->W; i++) {
        e->Rs[i] = Mat3();
        e->Ps[i] = e->Vs[i] = e->Bas[i] = e->Bgs[i] = Vec3();
        e->dt_buf[i].clear();
        e->acc_buf[i].clear();
        e->gyr_buf[i].clear();
        e->slot_valid[i] = false;
        e->slot_of[i] = i;
        e->flushed[i] = 0;
        e->sum_dt[i] = 0;
    }
    e->tic = Vec3();
    e->ric = Mat3();
    e->solver_flag = 0;
    e->first_imu = false;
    e->frame_count = 0;
    e->td = e->cfg.td;
    e->has_prior = false;
    e->prior_n = 0;
    e->prior_blocks.clear();
    e->feature.clear();
    e->failure_occur = false;
    e->all_image_frame.clear();
    e->tmp_pre.valid = false;
    e->initial_timestamp = 0;
    e->relocalization_info = false;
    e->drift_correct_r = Mat3();
    e->drift_correct_t = Vec3();
}

void process_imu(ve_estimator* e, double dt, const Vec3& acc, const Vec3& gyr) {
    if (!e->first_imu) {
        e->first_imu = true;
        e->acc_0 = acc;
        e->gyr_0 = gyr;
    }
    const int j = e->frame_count;
    if (!e->slot_valid[j]) init_slot(e, j, e->acc_0, e->gyr_0, e->Bas[j], e->Bgs[j]);
    if (j != 0) {
        e->dt_buf[j].push_back(dt);
        e->acc_buf[j].push_back(acc);
        e->gyr_buf[j].push_back(gyr);
        e->sum_dt[j] += dt;
        if (e->solver_flag == 0 && e->tmp_pre.valid) e->tmp_pre.push_back(dt, acc, gyr);  // tmp_pre_integration->push_back
        const Vec3 un_acc_0 = e->Rs[j] * (e->acc_0 - e->Bas[j]) - e->g;
        const Vec3 un_gyr = 0.5 * (e->gyr_0 + gyr) - e->Bgs[j];
        e->Rs[j] = e->Rs[j] * vb::deltaQ(un_gyr * dt).R();
        const Vec3 un_acc_1 = e->Rs[j] * (acc - e->Bas[j]) - e->g;
        const Vec3 un_acc = 0.5 * (un_acc_0 + un_acc_1);
        e->Ps[j] += dt * e->Vs[j] + 0.5 * dt * dt * un_acc;
        e->Vs[j] += dt * un_acc;
    }
    e->acc_0 = acc;
    e->gyr_0 = gyr;
}

bool initial_from_seed(ve_estimator* e) {
    for (int i = 0; i <= e->W; i++) {
        const SeedRow* s = nullptr;
        for (auto& c : e->seeds)
            if (std::fabs(c.t - e->Headers[i]) < 1e-6) s = &c;
        if (!s) return false;
    }
    for (int i = 0; i <= e->W; i++) {
        const SeedRow* s = nullptr;
        for (auto& c : e->seeds)
            if (std::fabs(c.t - e->Headers[i]) < 1e-6) s = &c;
        e->Ps[i] = s->P; e->Rs[i] = s->R; e->Vs[i] = s->V; e->Bas[i] = e->seed_ba; e->Bgs[i] = e->seed_bg;
    }
    for (int i = 0; i <= e->W; i++) {  // IntegrationBase::repropagate(Bas[i], Bgs[i])
        if (!e->slot_valid[i]) continue;
        const Vec3 la = e->lin_acc[i], lg = e->lin_gyr[i];
        init_slot(e, i, la, lg, e->Bas[i], e->Bgs[i]);
        e->sum_dt[i] = 0;
        for (double v : e->dt_buf[i]) e->sum_dt[i] += v;
        flush_frame(e, i);
    }
    for (auto& it : e->feature) it.estimated_depth = -1;
    triangulate(e);
    return true;
}

bool seeds_cover_window(const ve_estimator* e) {
    for (int i = 0; i <= e->W; i++) {
        bool found = false;
        for (auto& c : e->seeds)
            if (std::fabs(c.t - e->Headers[i]) < 1e-6) found = true;
        if (!found) return false;
    }
    return !e->seeds.empty();
}

// Estimator::initialStructure + visualInitialAlign (estimator.cpp:218-440).  The stages up to VisualIMUAlignment live in
// initial.cpp; this is the "change state" tail that writes the window.
bool initial_structure(ve_estimator* e) {
    namespace vi = vb::init;
    const int W = e->W;
    std::vector<vi::Track> tracks;
    tracks.reserve(e->feature.size());
    for (auto& it : e->feature) {
        vi::Track t;
        t.id = it.feature_id;
        t.start_frame = it.start_frame;
        for (auto& f : it.feature_per_frame) {
            t.xy.push_back(f.point.x);
            t.xy.push_back(f.point.y);
        }
        tracks.push_back(std::move(t));
    }
    const Mat3 RIC = e->RIC;
    const Vec3 TIC(e->cfg.tic[0], e->cfg.tic[1], e->cfg.tic[2]);
    std::vector<double> headers(e->Headers.begin(), e->Headers.begin() + W + 1), x;
    std::vector<Vec3> Bgs(e->Bgs.begin(), e->Bgs.begin() + W + 1);
    const vi::Result res = vi::initial_structure(e->all_image_frame, headers, tracks, RIC, TIC, e->cfg.g_norm, Bgs, x);
    e->init_l = res.l;
    e->init_iterations = res.sfm_iterations;
    e->init_cost = res.sfm_cost;
    if (res.code == vi::INIT_FAIL_SFM) e->marginalization_flag = 0;  // estimator.cpp:284
    if (res.code != vi::INIT_OK) {
        e->init_failures++;
        return false;
    }
    for (int i = 0; i <= W; i++) e->Bgs[i] = Bgs[i];
    // visualInitialAlign: change state
    auto frame_at = [&](double t) -> vi::ImageFrame& {
        for (auto& f : e->all_image_frame)
            if (f.t == t) return f;
        return e->all_image_frame.back();
    };
    for (int i = 0; i <= e->frame_count; i++) {
        vi::ImageFrame& f = frame_at(e->Headers[i]);
        e->Ps[i] = f.T;
        e->Rs[i] = f.R;
        f.is_key_frame = true;
    }
    for (auto& it : e->feature) it.estimated_depth = -1;
    // triangulate on the camera poses, no tic
    const Vec3 tic_keep = e->tic;
    e->tic = Vec3();
    e->ric = RIC;
    triangulate(e);
    e->tic = tic_keep;
    const double s = x.back();
    for (int i = 0; i <= W; i++) {  // pre_integrations[i]->repropagate(0, Bgs[i])
        if (!e->slot_valid[i]) continue;
        const Vec3 la = e->lin_acc[i], lg = e->lin_gyr[i];
        init_slot(e, i, la, lg, Vec3(), e->Bgs[i]);
        e->sum_dt[i] = 0;
        for (double v : e->dt_buf[i]) e->sum_dt[i] += v;
        flush_frame(e, i);
    }
    for (int i = e->frame_count; i >= 0; i--) e->Ps[i] = s * e->Ps[i] - e->Rs[i] * TIC - (s * e->Ps[0] - e->Rs[0] * TIC);
    int kv = -1;
    for (auto& f : e->all_image_frame)
        if (f.is_key_frame) {
            kv++;
            // the reference indexes the alignment vector with the key-frame counter (estimator.cpp:400-408)
            e->Vs[kv] = f.R * Vec3(x[3 * kv], x[3 * kv + 1], x[3 * kv + 2]);
        }
    for (auto& it : e->feature) {
        if (!usable(e, it)) continue;
        it.estimated_depth *= s;
    }
    Mat3 R0 = vi::g2R(res.g);
    const double yaw = vb::R2ypr(R0 * e->Rs[0]).x;
    R0 = vb::ypr2R(Vec3(-yaw, 0, 0)) * R0;
    e->g = R0 * res.g;
    for (int i = 0; i <= e->frame_count; i++) {
        e->Ps[i] = R0 * e->Ps[i];
        e->Rs[i] = R0 * e->Rs[i];
        e->Vs[i] = R0 * e->Vs[i];
    }
    e->init_scale = s;
    e->self_initialised = true;
    return true;
}

bool failure_detection(ve_estimator* e) {
    const int W = e->W;
    if (e->Bas[W].norm() > 2.5) return true;
    if (e->Bgs[W].norm() > 1.0) return true;
    const Vec3 tmp_P = e->Ps[W];
    if ((tmp_P - e->last_P).norm() > 5) return true;
    if (std::fabs(tmp_P.z - e->last_P.z) > 1) return true;
    return false;
}

// vector2double (estimator.cpp:486-528): packs the window into a states vector whose view `x` has room for its landmarks
void pack_states(ve_estimator* e, const vb::BaStates& x) {
    const int F = e->W + 1;
    for (int i = 0; i < F; i++) {
        const Quat q = Quat::FromR(e->Rs[i]);
        double* p = x.pose + 7 * i;
        p[0] = e->Ps[i].x; p[1] = e->Ps[i].y; p[2] = e->Ps[i].z; p[3] = q.x; p[4] = q.y; p[5] = q.z; p[6] = q.w;
        double* s = x.sb + 9 * i;
        s[0] = e->Vs[i].x; s[1] = e->Vs[i].y; s[2] = e->Vs[i].z;
        s[3] = e->Bas[i].x; s[4] = e->Bas[i].y; s[5] = e->Bas[i].z;
        s[6] = e->Bgs[i].x; s[7] = e->Bgs[i].y; s[8] = e->Bgs[i].z;
    }
    const Quat q = Quat::FromR(e->ric);
    x.ex[0] = e->tic.x; x.ex[1] = e->tic.y; x.ex[2] = e->tic.z; x.ex[3] = q.x; x.ex[4] = q.y; x.ex[5] = q.z; x.ex[6] = q.w;
    x.td[0] = e->td;
    int k = 0;
    for (auto& it : e->feature)
        if (usable(e, it)) x.lam[k++] = 1. / it.estimated_depth;
    for (int q7 = 0; q7 < 7; q7++) x.relo[q7] = e->relo_Pose[q7];
}

// Results of the device-side double2vector (ba_finish_kernel) -> Estimator members.
void unpack_results(ve_estimator* e, const double* out) {
    const int F = e->W + 1;
    const vb::BaOutLayout ol = vb::ba_out_layout(F, e->fr_L, e->fr_relo);
    std::memcpy(&e->last_state, out, sizeof(vb::SolverState));
    for (int i = 0; i < F; i++) {
        const double* o = out + ol.frames + vb::BA_OUT_FRAME * i;
        e->Ps[i] = Vec3(o[0], o[1], o[2]);
        std::memcpy(e->Rs[i].m, o + 3, 9 * sizeof(double));
        e->Vs[i] = Vec3(o[12], o[13], o[14]);
        e->Bas[i] = Vec3(o[15], o[16], o[17]);
        e->Bgs[i] = Vec3(o[18], o[19], o[20]);
    }
    const double* x = out + ol.ex;
    e->tic = Vec3(x[0], x[1], x[2]);
    std::memcpy(e->ric.m, x + 3, 9 * sizeof(double));
    if (e->cfg.estimate_td) e->td = x[12];
    const double* od = out + ol.depths;
    int k = 0;
    for (auto& it : e->feature) {  // FeatureManager::setDepth
        if (!usable(e, it)) continue;
        it.estimated_depth = od[k++];
        it.solve_flag = it.estimated_depth < 0 ? 2 : 1;
    }
    for (int i = 0; i < F; i++) {  // what the closing vector2double leaves in para_Pose (setReloFrame copies from it)
        const Quat q = Quat::FromR(e->Rs[i]);
        e->para_Pose[i] = {e->Ps[i].x, e->Ps[i].y, e->Ps[i].z, q.x, q.y, q.z, q.w};
    }
    if (e->fr_relo) {  // drift bookkeeping of double2vector (estimator.cpp:598-617); relo_r / relo_t come from the device
        const double* ro = out + ol.relo;
        Mat3 relo_r;
        std::memcpy(relo_r.m, ro, 9 * sizeof(double));
        const Vec3 relo_t(ro[9], ro[10], ro[11]);
        const double drift_correct_yaw = vb::R2ypr(e->prev_relo_r).x - vb::R2ypr(relo_r).x;
        e->drift_correct_r = vb::ypr2R(Vec3(drift_correct_yaw, 0, 0));
        e->drift_correct_t = e->prev_relo_t - e->drift_correct_r * relo_t;
        const int li = e->relo_frame_local_index;
        e->relo_relative_t = relo_r.T() * (e->Ps[li] - relo_t);
        e->relo_relative_q = Quat::FromR(relo_r.T() * e->Rs[li]);
        e->relo_relative_yaw = vb::normalize_angle(vb::R2ypr(e->Rs[li]).x - vb::R2ypr(relo_r).x);  // Utility::normalizeAngle
        e->relocalization_info = false;
        e->fr_relo = false;
        e->n_relo_solves++;
    }
}

struct MargHost {  // host side of one marginalisation plan
    bool run = false;
    std::vector<int> lms, col_lm;
    std::vector<PriorBlock> kept, shifted;
};

// The marginalisation branches of Estimator::optimization (estimator.cpp:826-999): everything but the arithmetic is
// known before the solve (which blocks are dropped, the column layout, the identities of the kept blocks).
int plan_marginalization(ve_estimator* e, vb::MargPlan& mp, MargHost& mh) {
    const int W = e->W, F = W + 1;
    const bool old = e->marginalization_flag == 0;
    auto prior_has = [&](int type, int index) {
        for (auto& b : e->prior_blocks)
            if (b.type == type && (type >= 2 || b.index == index)) return true;
        return false;
    };
    mh.run = false;
    if (!old && !(e->has_prior && prior_has(0, W - 1))) return VE_OK;
    std::vector<bool> t_pose(F, false), t_sb(F, false);
    bool t_ex = false, t_td = false;
    if (e->has_prior)
        for (auto& b : e->prior_blocks) {
            if (b.type == 0) t_pose[b.index] = true;
            else if (b.type == 1) t_sb[b.index] = true;
            else if (b.type == 2) t_ex = true;
            else t_td = true;
        }
    mp.use_imu = 0;
    if (old) {
        if (e->slot_valid[1] && e->sum_dt[1] < 10.0) {
            mp.use_imu = 1;
            t_pose[0] = t_sb[0] = t_pose[1] = t_sb[1] = true;
        }
        int li = -1;
        for (auto& it : e->feature) {
            if (!usable(e, it)) continue;
            ++li;
            if (it.start_frame != 0) continue;
            mh.lms.push_back(li);
            t_pose[0] = true;
            for (size_t k = 1; k < it.feature_per_frame.size(); k++) t_pose[k] = true;
            t_ex = true;
            if (e->cfg.estimate_td) t_td = true;
        }
    }
    // column layout: marginalised dense blocks, marginalised landmarks, kept blocks (canonical order)
    int pos = 0;
    for (int f = 0; f < vb::BA_MAX_FRAMES; f++) mp.col_pose[f] = mp.col_sb[f] = -1;
    mp.col_ex = mp.col_td = -1;
    const int drop_pose = old ? 0 : W - 1;
    if (t_pose[drop_pose]) { mp.col_pose[drop_pose] = pos; pos += 6; }
    if (old && t_sb[0]) { mp.col_sb[0] = pos; pos += 9; }
    mp.m_dense = pos;
    for (size_t k = 0; k < mh.lms.size(); k++) mh.col_lm.push_back(pos++);
    mp.n_lm = (int)mh.lms.size();
    const int m = pos;
    for (int f = 0; f < F; f++)
        if (t_pose[f] && mp.col_pose[f] < 0) { mp.col_pose[f] = pos; mh.kept.push_back({0, f, pos - m, 6}); pos += 6; }
    for (int f = 0; f < F; f++)
        if (t_sb[f] && mp.col_sb[f] < 0) { mp.col_sb[f] = pos; mh.kept.push_back({1, f, pos - m, 9}); pos += 9; }
    if (t_ex) { mp.col_ex = pos; mh.kept.push_back({2, 0, pos - m, 6}); pos += 6; }
    if (t_td) { mp.col_td = pos; mh.kept.push_back({3, 0, pos - m, 1}); pos += 1; }
    mp.P = pos;
    mp.n = pos - m;
    if (mp.n > e->nmax || mp.P > (int)vb::ba_marg_layout(e->nmax, e->Lmax).P || mp.m_dense == 0 || (int)mh.kept.size() > vb::BA_MAX_PRIOR_BLOCKS) {
        e->err = "marginalisation system larger than the configured capacity";
        return VE_ERR_CAPACITY;
    }
    // identities of the kept blocks after the slide (addr_shift, estimator.cpp:913-925 / :969-990)
    for (auto nbk : mh.kept) {
        if (nbk.type <= 1) {
            if (old) nbk.index -= 1;
            else if (nbk.index == W) nbk.index = W - 1;
        }
        mh.shifted.push_back(nbk);
    }
    mh.run = true;
    return VE_OK;
}

// Builds this member's part of the frame: the input block (jobs, samples, observation table, states, marginalisation
// lists) in the pinned arena and its descriptor.  `solve` = the window is optimised this frame.
int stage_frame(ve_estimator* e, bool solve) {
    ve_batch* b = e->batch;
    vb::BaSeq& q = b->h_seq[e->member];
    const int W = e->W, F = W + 1;
    q.active = 0;
    q.do_marg = 0;
    q.n_jobs = 0;
    q.sqrt_mask = 0;
    e->fr_marg = false;
    int L = 0, M = 0;
    vb::MargPlan mp{};
    MargHost mh;
    std::vector<int> relo_match;  // per landmark: index of its relocalisation match in match_points, or -1
    e->fr_relo = false;
    if (solve) {
        for (int f = 0; f <= W; f++) flush_frame(e, f);
        q.sqrt_mask = refresh_sqrt_mask(e);
        // the solver's column tables hold BA_MAX_D entries (W = 22 with extrinsic and td): a relocalisation block that would not
        // fit is left out (only possible at the largest window with both optional blocks live)
        const bool relo = e->relocalization_info && 15 * F + 6 * (e->cfg.estimate_extrinsic ? 1 : 0) + (e->cfg.estimate_td ? 1 : 0) + 6 <= vb::BA_MAX_D;
        const size_t n_match = e->match_points.size() / 3;
        size_t retrive_feature_index = 0;
        int n_relo = 0;
        for (auto& it : e->feature) {
            if (!usable(e, it)) continue;
            if (L >= e->Lmax || M + (int)it.feature_per_frame.size() + 1 > e->Mmax) {
                e->err = "feature capacity (max_features) exceeded";  // NUM_OF_F overflow is silent in the reference (estimator.h:111)
                return VE_ERR_CAPACITY;
            }
            M += (int)it.feature_per_frame.size() - 1;
            L++;
            if (relo) {  // the walk of estimator.cpp:777-797 (bounded: the reference runs off match_points' end)
                int hit = -1;
                if (it.start_frame <= e->relo_frame_local_index) {
                    while (retrive_feature_index < n_match && (int)e->match_points[3 * retrive_feature_index + 2] < it.feature_id)
                        retrive_feature_index++;
                    if (retrive_feature_index < n_match && (int)e->match_points[3 * retrive_feature_index + 2] == it.feature_id) {
                        hit = (int)retrive_feature_index++;
                        n_relo++;
                        M++;
                    }
                }
                relo_match.push_back(hit);
            }
        }
        // No matched landmark: Ceres drops a parameter block without residuals from the program, so the solve is the plain one;
        // the message is consumed (relo_Pose, hence the drift outputs, stay as they are).
        e->fr_relo = relo && n_relo > 0;
        if (relo && n_relo == 0) e->relocalization_info = false;
        e->n_relo_factors = n_relo;
        const int rc = plan_marginalization(e, mp, mh);
        if (rc) return rc;
    }
    const size_t n_jobs = e->jobs.size(), n_rec = e->job_samples.size() / 7;
    if (!solve && n_jobs == 0) return VE_OK;
    const size_t n_lm = mh.lms.size();
    const vb::BaInLayout il = vb::ba_in_layout(W, n_jobs, n_rec, L, M, n_lm, solve);
    ve_batch::Group& grp = b->groups[e->member / b->members_per_group];
    const size_t rel = grp.in_used.fetch_add(il.total);
    const size_t base = grp.in_base + rel;
    if (rel + il.total > grp.in_cap) {
        e->err = "batch input arena exhausted";
        return VE_ERR_CAPACITY;
    }
    // the block's arrays in the pinned arena (filled here) and in its device copy (what the kernels read)
    const vb::BaInPtrs hin = vb::ba_in_bind(b->h_in + base, il), din = vb::ba_in_bind(b->d_in + base, il);
    e->h2d_bytes = il.total + sizeof(vb::BaSeq);
    // pre-integration jobs
    if (n_jobs) std::memcpy(hin.jobs, e->jobs.data(), n_jobs * sizeof(vb::PreintJob));
    if (n_rec) std::memcpy(hin.samples, e->job_samples.data(), n_rec * 7 * sizeof(double));
    q.n_jobs = (int)n_jobs;
    q.jobs = din.jobs;
    q.samples = din.samples;
    q.noise[0] = e->cfg.acc_n; q.noise[1] = e->cfg.gyr_n; q.noise[2] = e->cfg.acc_w; q.noise[3] = e->cfg.gyr_w;
    q.p.preint = e->d_preint;
    e->jobs.clear();
    e->job_samples.clear();
    if (!solve) return VE_OK;

    // ---- observation table grouped by landmark (Estimator::optimization's problem assembly, estimator.cpp:670-801)
    int *lm_anchor = hin.lm_anchor, *lm_start = hin.lm_start, *ob_frame = hin.ob_frame, *imu_slot = hin.imu_slot, *lm_relo = hin.lm_relo;
    double *lm_pts = hin.lm_pts, *lm_vel = hin.lm_vel, *lm_td = hin.lm_td, *lm_row = hin.lm_row;
    double *ob_pts = hin.ob_pts, *ob_vel = hin.ob_vel, *ob_td = hin.ob_td, *ob_row = hin.ob_row;
    int l = 0, m = 0;
    for (auto& it : e->feature) {
        if (!usable(e, it)) continue;
        const FeaturePerFrame& f0 = it.feature_per_frame[0];
        lm_anchor[l] = it.start_frame;
        lm_start[l] = m;
        lm_pts[2 * l] = f0.point.x; lm_pts[2 * l + 1] = f0.point.y;
        lm_vel[2 * l] = f0.vx; lm_vel[2 * l + 1] = f0.vy;
        lm_td[l] = f0.cur_td;
        lm_row[l] = f0.v;
        for (size_t k = 1; k < it.feature_per_frame.size(); k++) {
            const FeaturePerFrame& fj = it.feature_per_frame[k];
            ob_frame[m] = it.start_frame + (int)k;
            ob_pts[2 * m] = fj.point.x; ob_pts[2 * m + 1] = fj.point.y;
            ob_vel[2 * m] = fj.vx; ob_vel[2 * m + 1] = fj.vy;
            ob_td[m] = fj.cur_td;
            ob_row[m] = fj.v;
            m++;
        }
        lm_relo[l] = 0;
        if (e->fr_relo && relo_match[l] >= 0) {  // ProjectionFactor(pts_i, pts_j = match) against relo_Pose: the row behind the track
            const double* mpt = &e->match_points[3 * (size_t)relo_match[l]];
            ob_frame[m] = -1;
            ob_pts[2 * m] = mpt[0]; ob_pts[2 * m + 1] = mpt[1];
            ob_vel[2 * m] = 0; ob_vel[2 * m + 1] = 0;
            ob_td[m] = f0.cur_td;
            ob_row[m] = 0;
            lm_relo[l] = 1;
            m++;
        }
        l++;
    }
    lm_start[L] = M;
    for (int k = 0; k < W; k++) imu_slot[k] = (e->sum_dt[k + 1] > 10.0 || !e->slot_valid[k + 1]) ? -1 : e->slot_of[k + 1];
    pack_states(e, vb::states_view(hin.states, F, L));

    vb::BaProblem& p = q.p;
    vb::BaDims& d = p.dims;
    d.W = W;
    d.L = L;
    d.M = M;
    d.est_ex = e->cfg.estimate_extrinsic ? 1 : 0;
    d.est_td = e->cfg.estimate_td ? 1 : 0;
    d.col_sb = 6 * F;
    d.col_ex = d.est_ex ? 15 * F : -1;
    d.col_td = d.est_td ? 15 * F + 6 * d.est_ex : -1;
    d.D = 15 * F + 6 * d.est_ex + d.est_td;
    d.col_relo = -1;
    if (e->fr_relo) {  // relo_Pose: one more pose block behind every other column
        d.col_relo = d.D;
        d.D += 6;
    }
    d.sqrt_info_vis = e->cfg.focal_length / 1.5;
    d.tr_over_row = e->cfg.tr / e->cfg.row;
    d.half_row = e->cfg.row / 2;
    d.G[0] = 0; d.G[1] = 0; d.G[2] = e->cfg.g_norm;
    p.x[0] = vb::states_view(din.states, F, L);
    p.x[1] = vb::states_view(e->d_states1, F, L);
    const bool wide = d.est_ex || d.est_td;
    d.oj = wide ? vb::OJ_FULL : vb::OJ_BASE;
    d.lw = wide ? vb::LW_FULL : vb::LW_BASE;
    const vb::BaAccLayout al = vb::ba_acc_layout(W, e->Lmax, e->Mmax, e->D);
    for (int k = 0; k < 2; k++) {  // sized for the widest records; the kernels index with dims.oj / dims.lw
        double* a = e->d_acc[k];
        p.acc[k] = vb::BaAccum{a + al.obsJ, a + al.lmW, a + al.imuJ, a + al.gpr, a + al.gp, a + al.cost};
    }
    p.lm_anchor = din.lm_anchor;
    p.lm_start = din.lm_start;
    p.ob_frame = din.ob_frame;
    p.imu_slot = din.imu_slot;
    p.lm_relo = din.lm_relo;
    p.lm_pts = din.lm_pts;
    p.lm_vel = din.lm_vel;
    p.lm_td = din.lm_td;
    p.lm_row = din.lm_row;
    p.ob_pts = din.ob_pts;
    p.ob_vel = din.ob_vel;
    p.ob_td = din.ob_td;
    p.ob_row = din.ob_row;
    // current prior
    vb::BaPrior& pr = p.prior;
    pr = vb::BaPrior{};
    vb::BaSeq* dq = b->d_seq + e->member;
    const vb::BaPriorLayout pl = vb::ba_prior_layout(e->nmax);
    if (e->has_prior) {
        pr.n = e->prior_n;
        pr.nblocks = (int)e->prior_blocks.size();
        for (int k = 0; k < pr.nblocks; k++) {
            q.prior_type[k] = e->prior_blocks[k].type;
            q.prior_index[k] = e->prior_blocks[k].index;
            q.prior_off[k] = e->prior_blocks[k].off;
        }
        pr.type = dq->prior_type;  // addresses inside the device copy of this descriptor
        pr.index = dq->prior_index;
        pr.off = dq->prior_off;
        const double* a = e->d_prior[e->prior_buf];
        pr.A = a + pl.A;
        pr.g0 = a + pl.g0;
        pr.c0 = a + pl.c0;
        pr.x0 = a + pl.x0;
    }
    p.S = e->d_S;
    p.Spk = e->d_Spk;
    p.Hfull = e->d_Hfull;
    p.gred = e->d_gred;
    const vb::BaVecLayout vl = vb::ba_vec_layout(e->D, e->Lmax);
    p.scale = e->d_vec + vl.scale;
    p.diag = e->d_vec + vl.diag;
    p.grad = e->d_vec + vl.grad;
    p.gn = e->d_vec + vl.gn;
    p.work = e->d_work;
    p.st = &dq->st;
    vb::SolverState& st = q.st;
    std::memset(&st, 0, sizeof(st));
    st.max_iterations = e->cfg.num_iterations;
    st.first = 1;
    st.radius = 1e4;
    st.mu = 1e-8;
    // ---- double2vector inputs and the output block
    vb::FinishPlan& fp = q.fin;
    Vec3 origin_R0 = vb::R2ypr(e->Rs[0]);
    Vec3 origin_P0 = e->Ps[0];
    if (e->failure_occur) {
        origin_R0 = vb::R2ypr(e->last_R0);
        origin_P0 = e->last_P0;
        e->failure_occur = false;
    }
    fp.origin_ypr[0] = origin_R0.x; fp.origin_ypr[1] = origin_R0.y; fp.origin_ypr[2] = origin_R0.z;
    fp.origin_P0[0] = origin_P0.x; fp.origin_P0[1] = origin_P0.y; fp.origin_P0[2] = origin_P0.z;
    std::memcpy(fp.Rs0, e->Rs[0].m, sizeof(fp.Rs0));
    const size_t out_doubles = vb::ba_out_layout(F, L, e->fr_relo).total;
    const size_t orel = grp.out_used.fetch_add(vb::ba_out_reserve(F, L, e->fr_relo));
    const size_t obase = grp.out_base + orel;
    if (orel + out_doubles > grp.out_cap) {
        e->err = "batch output arena exhausted";
        return VE_ERR_CAPACITY;
    }
    e->out_off = obase;
    e->d2h_bytes = out_doubles * sizeof(double);
    fp.out = b->d_out + obase;
    fp.n_kept = 0;
    fp.x0_out = nullptr;
    // ---- marginalisation
    if (mh.run) {
        for (size_t k = 0; k < n_lm; k++) {
            hin.marg_lms[k] = mh.lms[k];
            hin.marg_col_lm[k] = mh.col_lm[k];
        }
        mp.lms = din.marg_lms;
        mp.col_lm = din.marg_col_lm;
        const vb::BaMargLayout ml = vb::ba_marg_layout(e->nmax, e->Lmax);
        mp.Am = e->d_marg + ml.Am;
        mp.bm = e->d_marg + ml.bm;
        mp.Araw = e->d_marg + ml.Araw;
        mp.graw = e->d_marg + ml.graw;
        mp.Wglobal = e->d_marg + ml.Wglobal;
        mp.w_in_global = b->w_in_global;  // fixed at batch creation
        const int nb = e->prior_buf ^ 1;
        mp.Aout = e->d_prior[nb] + pl.A;  // written with leading dimension n (dense n x n at the front of the buffer)
        mp.gout = e->d_prior[nb] + pl.g0;
        mp.cout = e->d_prior[nb] + pl.c0;
        fp.n_kept = (int)mh.kept.size();
        for (int k = 0; k < fp.n_kept; k++) {
            fp.kept_type[k] = mh.kept[k].type;
            fp.kept_index[k] = mh.kept[k].index;
        }
        fp.x0_out = e->d_prior[nb] + pl.x0;
        q.mp = mp;
        q.do_marg = 1;
        e->fr_marg = true;
        e->marg_Araw = mp.Araw;
        e->marg_graw = mp.graw;
        e->marg_n = mp.n;
        // the new prior replaces the old one for every later frame
        e->prior_blocks = mh.shifted;
        e->prior_n = mp.n;
        e->prior_buf = nb;
        e->has_prior = true;
    }
    q.active = 1;
    e->fr_L = L;
    e->last_landmarks = L;
    e->last_visual = M - (e->fr_relo ? e->n_relo_factors : 0);  // f_m_cnt counts the window's factors only (estimator.cpp:766)
    return VE_OK;
}

void slide_window_old(ve_estimator* e) {
    if (e->solver_flag == 1) {
        const Mat3 R0 = e->back_R0 * e->ric, R1 = e->Rs[0] * e->ric;
        const Vec3 P0 = e->back_P0 + e->back_R0 * e->tic, P1 = e->Ps[0] + e->Rs[0] * e->tic;
        remove_back_shift_depth(e, R0, P0, R1, P1);
    } else
        remove_back(e);
}

void slide_window(ve_estimator* e) {
    const int W = e->W;
    if (e->marginalization_flag == 0) {
        const double t_0 = e->Headers[0];
        e->back_R0 = e->Rs[0];
        e->back_P0 = e->Ps[0];
        if (e->frame_count == W) {
            // all_image_frame.erase(begin, t_0] (estimator.cpp:1034-1051)
            e->all_image_frame.erase(std::remove_if(e->all_image_frame.begin(), e->all_image_frame.end(),
                                                    [&](const vb::init::ImageFrame& f) { return f.t <= t_0; }),
                                     e->all_image_frame.end());
            const int slot0 = e->slot_of[0];
            for (int i = 0; i < W; i++) {
                std::swap(e->Rs[i], e->Rs[i + 1]);
                e->slot_of[i] = e->slot_of[i + 1];
                { bool t = e->slot_valid[i]; e->slot_valid[i] = e->slot_valid[i + 1]; e->slot_valid[i + 1] = t; }
                std::swap(e->flushed[i], e->flushed[i + 1]);
                std::swap(e->sum_dt[i], e->sum_dt[i + 1]);
                std::swap(e->lin_acc[i], e->lin_acc[i + 1]);
                std::swap(e->lin_gyr[i], e->lin_gyr[i + 1]);
                e->dt_buf[i].swap(e->dt_buf[i + 1]);
                e->acc_buf[i].swap(e->acc_buf[i + 1]);
                e->gyr_buf[i].swap(e->gyr_buf[i + 1]);
                e->Headers[i] = e->Headers[i + 1];
                std::swap(e->Ps[i], e->Ps[i + 1]);
                std::swap(e->Vs[i], e->Vs[i + 1]);
                std::swap(e->Bas[i], e->Bas[i + 1]);
                std::swap(e->Bgs[i], e->Bgs[i + 1]);
            }
            e->slot_of[W] = slot0;
            e->Headers[W] = e->Headers[W - 1];
            e->Ps[W] = e->Ps[W - 1]; e->Vs[W] = e->Vs[W - 1]; e->Rs[W] = e->Rs[W - 1];
            e->Bas[W] = e->Bas[W - 1]; e->Bgs[W] = e->Bgs[W - 1];
            init_slot(e, W, e->acc_0, e->gyr_0, e->Bas[W], e->Bgs[W]);
            e->dt_buf[W].clear(); e->acc_buf[W].clear(); e->gyr_buf[W].clear();
            slide_window_old(e);
        }
    } else if (e->frame_count == W) {
        const int fc = e->frame_count;
        for (size_t i = 0; i < e->dt_buf[fc].size(); i++) {
            e->dt_buf[fc - 1].push_back(e->dt_buf[fc][i]);
            e->acc_buf[fc - 1].push_back(e->acc_buf[fc][i]);
            e->gyr_buf[fc - 1].push_back(e->gyr_buf[fc][i]);
            e->sum_dt[fc - 1] += e->dt_buf[fc][i];
        }
        flush_frame(e, fc - 1);  // pre_integrations[frame_count - 1]->push_back(...)
        e->Headers[fc - 1] = e->Headers[fc];
        e->Ps[fc - 1] = e->Ps[fc]; e->Vs[fc - 1] = e->Vs[fc]; e->Rs[fc - 1] = e->Rs[fc];
        e->Bas[fc - 1] = e->Bas[fc]; e->Bgs[fc - 1] = e->Bgs[fc];
        init_slot(e, W, e->acc_0, e->gyr_0, e->Bas[W], e->Bgs[W]);
        e->dt_buf[W].clear(); e->acc_buf[W].clear(); e->gyr_buf[W].clear();
        remove_front(e, fc);
    }
}

void remove_failures(ve_estimator* e) {
    e->feature.erase(std::remove_if(e->feature.begin(), e->feature.end(), [](const FeaturePerId& f) { return f.solve_flag == 2; }),
                     e->feature.end());
}

// Estimator::processImage up to the point where the window is handed to the solver (estimator.cpp:120-217).
int prepare_frame(ve_estimator* e, int n, const int* ids, const double* xyz_uv_vel, double stamp) {
    e->h2d_bytes = e->d2h_bytes = 0;
    e->stage = STAGE_DONE;
    std::vector<int> order(n);
    for (int i = 0; i < n; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ids[a] < ids[b]; });
    e->marginalization_flag = add_feature_check_parallax(e, n, order.data(), ids, xyz_uv_vel, e->td) ? 0 : 1;
    e->Headers[e->frame_count] = stamp;
    const int W = e->W;
    bool solve = false;
    if (e->solver_flag == 0) {
        // ImageFrame imageframe(image, stamp); imageframe.pre_integration = tmp_pre_integration; new tmp_pre_integration
        vb::init::ImageFrame fr;
        fr.t = stamp;
        fr.ids.resize(n);
        fr.xy.resize(2 * (size_t)n);
        for (int k = 0; k < n; k++) {
            fr.ids[k] = ids[order[k]];
            fr.xy[2 * k] = xyz_uv_vel[7 * order[k]];
            fr.xy[2 * k + 1] = xyz_uv_vel[7 * order[k] + 1];
        }
        fr.pre = e->tmp_pre;
        e->all_image_frame.push_back(std::move(fr));
        e->tmp_pre.start(e->acc_0, e->gyr_0, e->Bas[e->frame_count], e->Bgs[e->frame_count]);
        if (e->ex_calib_pending && e->frame_count != 0) {  // CalibrationExRotation (estimator.cpp:140-156)
            const int fc = e->frame_count;
            std::vector<double> corres;  // f_manager.getCorresponding(frame_count - 1, frame_count)
            for (auto& it : e->feature)
                if (it.start_frame <= fc - 1 && it.endFrame() >= fc) {
                    const Vec3 &a = it.feature_per_frame[fc - 1 - it.start_frame].point, &b2 = it.feature_per_frame[fc - it.start_frame].point;
                    corres.push_back(a.x); corres.push_back(a.y); corres.push_back(b2.x); corres.push_back(b2.y);
                }
            Mat3 calib_ric;
            // pre_integrations[frame_count]->delta_q: the samples since the previous image, i.e. the pre-integration just stored
            const vb::init::Preint& pre = e->all_image_frame.back().pre;
            if (pre.valid && e->initial_ex_rotation.calibrate(corres, pre.dq, W, calib_ric)) {
                e->ric = calib_ric;
                e->RIC = calib_ric;
                e->ex_calib_pending = false;  // ESTIMATE_EXTRINSIC = 1
            }
        }
        if (e->frame_count == W) {
            bool result = false;
            if (e->ex_calib_pending) {
                // no initialisation while the rotation is unknown (estimator.cpp:163)
            } else if (seeds_cover_window(e)) {
                result = initial_from_seed(e);
                e->self_initialised = false;
            } else if (stamp - e->initial_timestamp > 0.1) {
                result = initial_structure(e);
                e->initial_timestamp = stamp;
            }
            if (result) {
                e->solver_flag = 1;
                e->stage = STAGE_INIT_SOLVE;
                solve = true;
                e->all_image_frame.clear();  // only read while INITIAL
                e->tmp_pre.valid = false;
            } else
                slide_window(e);
        } else
            e->frame_count++;
    } else {
        e->stage = STAGE_RUN_SOLVE;
        solve = true;
    }
    if (solve) triangulate(e);  // solveOdometry (estimator.cpp:473-484)
    const int rc = stage_frame(e, solve);
    if (rc) e->stage = STAGE_DONE;
    return rc;
}

// The rest of processImage once the solve's results are on the host.
void finish_frame(ve_estimator* e) {
    if (e->stage == STAGE_DONE) return;
    const int W = e->W;
    unpack_results(e, e->batch->h_out + e->out_off);
    e->n_solves++;
    if (e->stage == STAGE_RUN_SOLVE && failure_detection(e)) {
        e->failure_occur = true;
        clear_state(e);
        set_parameter(e);
        e->n_reboots++;
        e->stage = STAGE_DONE;
        return;
    }
    slide_window(e);
    remove_failures(e);
    e->last_R = e->Rs[W]; e->last_P = e->Ps[W]; e->last_R0 = e->Rs[0]; e->last_P0 = e->Ps[0];
    e->stage = STAGE_DONE;
}

struct FrameMsg {
    int active, n;
    const int* ids;
    const double* obs;
    double stamp;
};

// One frame of the batch: members with a message take part, the others idle.
int batch_process(ve_batch* b, const FrameMsg* msgs, int* status_out) {
    VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaSetDevice(b->cfg.device));
    const int S = b->S;
    static const bool trace = std::getenv("VINSB200_TRACE") != nullptr;
    const auto t0 = std::chrono::steady_clock::now();
    auto since = [&](std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); };
    for (int g = 0; g < b->G; g++) {
        b->groups[g].in_used.store(0);
        b->groups[g].out_used.store(0);
    }
    b->last_launches = 0;
    b->pool->run(S, [&](int k) {
        ve_estimator* e = b->members[k].get();
        vb::BaSeq& q = b->h_seq[k];
        q.active = q.do_marg = q.n_jobs = 0;
        q.sqrt_mask = 0;
        e->status = VE_OK;
        e->stage = STAGE_DONE;
        if (msgs[k].active) {
            e->status = prepare_frame(e, msgs[k].n, msgs[k].ids, msgs[k].obs, msgs[k].stamp);
            if (e->status != VE_OK) q.active = q.do_marg = 0;
        }
    });
    const double t_prepare = since(t0);
    const auto t1 = std::chrono::steady_clock::now();
    b->marg_timing_valid = false;
    b->last_ms[0] = b->last_ms[1] = b->last_ms[2] = b->last_ms[3] = 0;
    for (int g = 0; g < b->G; g++) {  // enqueue every group's chain; nothing is waited for inside this loop
        ve_batch::Group& grp = b->groups[g];
        grp.waits_results = grp.has_marg = false;
        vb::BatchShape sh{};
        sh.S = grp.count;
        sh.W = b->cfg.window_size;
        sh.D = 0;  // the largest reduced system of this frame (a relocalisation pose adds 6 columns to a member)
        sh.max_iterations = b->cfg.num_iterations;
        sh.est_ex = b->cfg.estimate_extrinsic ? 1 : 0;
        sh.est_td = b->cfg.estimate_td ? 1 : 0;
        sh.w_in_global = b->w_in_global;
        for (int k = grp.first; k < grp.first + grp.count; k++) {
            const vb::BaSeq& q = b->h_seq[k];
            if (q.n_jobs) sh.any_jobs = 1;
            if (!q.active) continue;
            sh.any_active = 1;
            sh.max_L = std::max(sh.max_L, q.p.dims.L);
            sh.D = std::max(sh.D, q.p.dims.D);
            if (q.p.dims.col_relo >= 0) sh.any_relo = 1;
            if (q.do_marg) {
                sh.any_marg = 1;
                sh.max_n_lm = std::max(sh.max_n_lm, q.mp.n_lm);
                sh.max_md = std::max(sh.max_md, q.mp.m_dense);
                sh.max_n = std::max(sh.max_n, q.mp.n);
                sh.max_P = std::max(sh.max_P, q.mp.P);
            }
        }
        if (!sh.any_jobs && !sh.any_active) continue;
        if (sh.any_marg) {  // reduced system of the marginalisation in shared memory whenever this frame's sizes fit
            sh.w_in_global = vb::marg_w_in_global(sh.max_md, sh.max_n);
            for (int k = grp.first; k < grp.first + grp.count; k++) b->h_seq[k].mp.w_in_global = sh.w_in_global;
        }
        vb::BaSeq* dq = b->d_seq + grp.first;
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaMemcpyAsync(dq, b->h_seq + grp.first, sizeof(vb::BaSeq) * grp.count, cudaMemcpyHostToDevice, grp.stream));
        const size_t in_bytes = std::min(grp.in_used.load(), grp.in_cap);
        if (in_bytes) VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaMemcpyAsync(b->d_in + grp.in_base, b->h_in + grp.in_base, in_bytes, cudaMemcpyHostToDevice, grp.stream));
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventRecord(grp.ev[0], grp.stream));
        vb::launch_preint_jobs(dq, sh, grp.stream, &b->last_launches, &b->prof);
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventRecord(grp.ev[1], grp.stream));
        vb::launch_ba_solve(dq, sh, grp.stream, &b->last_launches, &b->prof);
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventRecord(grp.ev[2], grp.stream));
        if (sh.any_active) {  // results travel on the copy stream while the marginalisation already runs
            VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaStreamWaitEvent(grp.copy_stream, grp.ev[2], 0));
            const size_t out_doubles = std::min(grp.out_used.load(), grp.out_cap);
            VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaMemcpyAsync(b->h_out + grp.out_base, b->d_out + grp.out_base, sizeof(double) * out_doubles, cudaMemcpyDeviceToHost,
                                    grp.copy_stream));
            VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventRecord(grp.ev[4], grp.copy_stream));
            grp.waits_results = true;
        } else {
            // jobs only: the input arena must not be rewritten before the copy has been consumed
            VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventRecord(grp.ev[4], grp.stream));
            grp.waits_results = true;
        }
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventRecord(grp.ev[5], grp.stream));
        vb::launch_marginalize(dq, sh, grp.stream, &b->last_launches, &b->prof);
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventRecord(grp.ev[3], grp.stream));
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaGetLastError());
        grp.has_marg = sh.any_marg != 0;
    }
    const double t_launch = since(t1);
    const auto t2 = std::chrono::steady_clock::now();
    for (int g = 0; g < b->G; g++) {
        ve_batch::Group& grp = b->groups[g];
        if (!grp.waits_results) continue;
        VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaEventSynchronize(grp.ev[4]));
        if (g == 0) {
            float t = 0;
            if (cudaEventElapsedTime(&t, grp.ev[0], grp.ev[1]) == cudaSuccess) b->last_ms[0] = t;
            if (cudaEventElapsedTime(&t, grp.ev[1], grp.ev[2]) == cudaSuccess) b->last_ms[1] = t;
            if (cudaEventElapsedTime(&t, grp.ev[0], grp.ev[2]) == cudaSuccess) b->last_ms[3] = t;
            b->marg_timing_valid = grp.has_marg;
        }
    }
    const double t_wait = since(t2);
    const auto t3 = std::chrono::steady_clock::now();
    b->pool->run(S, [&](int k) { finish_frame(b->members[k].get()); });
    if (trace) std::fprintf(stderr, "[ve_batch] prepare %.3f launch %.3f wait %.3f finish %.3f ms (S=%d)\n", t_prepare, t_launch, t_wait, since(t3), S);
    if (status_out)
        for (int k = 0; k < S; k++) status_out[k] = b->members[k]->status;
    return vb::roll_up(b, VE_OK);
}

int config_valid(const ve_config* cfg) {
    if (cfg->window_size < 3 || cfg->window_size + 1 > vb::BA_MAX_FRAMES || cfg->window_size + 1 > vb::BA_MAX_OBS_PER_LM ||
        cfg->max_features < 8 || cfg->num_iterations < 1 || cfg->estimate_extrinsic > 2 || cfg->estimate_extrinsic < 0)
        return 0;
    // work arrays of the single-CTA solvers: prior of 6 W + 9 + 6 + 1 parameters, reduced system of 15 (W + 1) + 7
    // columns (above W = 13 the reduced systems move from shared to global memory)
    if (6 * cfg->window_size + 16 > vb::BA_MAX_PRIOR_N || 15 * (cfg->window_size + 1) + 7 > vb::BA_MAX_D) return 0;
    return 1;
}

// Creates member k and appends it to the batch.
int create_member(ve_batch* b, int k) {
    std::unique_ptr<ve_estimator> e(new ve_estimator());
    e->cfg = b->cfg;
    e->batch = b;
    e->member = k;
    e->W = b->cfg.window_size;
    const int W = e->W, F = W + 1;
    e->Ps.resize(F); e->Vs.resize(F); e->Bas.resize(F); e->Bgs.resize(F); e->Rs.resize(F);
    e->Headers.assign(F, 0.0);
    e->para_Pose.assign(F, std::array<double, 7>{0, 0, 0, 0, 0, 0, 1});
    std::memcpy(e->RIC.m, b->cfg.ric, sizeof(e->RIC.m));
    e->ex_calib_pending = b->cfg.estimate_extrinsic == 2;
    e->dt_buf.resize(F); e->acc_buf.resize(F); e->gyr_buf.resize(F);
    e->slot_of.resize(F); e->slot_valid.assign(F, false); e->flushed.assign(F, 0); e->sum_dt.assign(F, 0.0);
    e->lin_acc.resize(F); e->lin_gyr.resize(F); e->sqrt_dirty.assign(F, true);
    e->Lmax = b->cfg.max_features;
    e->Mmax = b->cfg.max_features * (W + 1);  // + one relocalisation match per landmark
    e->D = 15 * F + 6 + 1 + 6;               // ex, td and a relocalisation pose on top of the window
    e->nmax = 6 * F + 9 * 2 + 6 + 1;
    clear_state(e.get());
    set_parameter(e.get());
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_preint.alloc(F));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_states1.alloc(vb::ba_states_layout(F, e->Lmax).total));
    for (int k2 = 0; k2 < 2; k2++) {
        VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_acc[k2].alloc(vb::ba_acc_layout(W, e->Lmax, e->Mmax, e->D).total));
        VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_prior[k2].alloc(vb::ba_prior_layout(e->nmax).total));
    }
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_S.alloc((size_t)e->D * e->D));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_Spk.alloc(vb::ba_spk_doubles(e->D)));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_Hfull.alloc((size_t)e->D * e->D));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_gred.alloc(e->D));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_vec.alloc(vb::ba_vec_layout(e->D, e->Lmax).total));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_work.alloc(vb::ba_work_layout(e->D, e->Lmax).total));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, e->d_marg.alloc(vb::ba_marg_layout(e->nmax, e->Lmax).total));
    b->members.push_back(std::move(e));
    return VE_OK;
}

}  // namespace

extern "C" {

int ve_batch_create(const ve_config* cfg, int n, ve_batch** out) {
    if (!cfg || !out || n < 1 || n > 4096) return VE_ERR_INVALID;
    *out = nullptr;
    if (!config_valid(cfg)) return VE_ERR_INVALID;
    if (!vb::device_available(cfg->device)) return VE_ERR_NO_DEVICE;
    std::unique_ptr<ve_batch, void (*)(ve_batch*)> b(new ve_batch(), ve_batch_destroy);
    b->cfg = *cfg;
    b->S = n;
    VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaSetDevice(cfg->device));
    // launch groups: VINSB200_BATCH_GROUPS overrides the default (two groups for batches of 32 members and more)
    // measured on an H100 SXM (400 W limit), 64 members, two alternating runs each: 1 group 6.50 / 6.55 k, 2 groups
    // 6.78 / 5.91 k, 3 groups 6.71 / 6.37 k, 4 groups 6.89 / 6.69 k frames/s, i.e. within the run-to-run spread
    int G = n >= 32 ? 2 : 1;
    if (const char* env = std::getenv("VINSB200_BATCH_GROUPS")) G = std::atoi(env);
    G = std::max(1, std::min(G, n));
    b->G = G;
    b->members_per_group = (n + G - 1) / G;
    b->G = G = (n + b->members_per_group - 1) / b->members_per_group;
    b->groups.reset(new ve_batch::Group[G]);
    for (int g = 0; g < G; g++) {
        ve_batch::Group& grp = b->groups[g];
        grp.first = g * b->members_per_group;
        grp.count = std::min(b->members_per_group, n - grp.first);
        VB_CUDA_CHECK(b, VE_ERR_CUDA, grp.stream.create());
        VB_CUDA_CHECK(b, VE_ERR_CUDA, grp.copy_stream.create());
        for (auto& ev : grp.ev) VB_CUDA_CHECK(b, VE_ERR_CUDA, ev.create());
    }
    for (int k = 0; k < n; k++) {
        const int rc = create_member(b.get(), k);
        if (rc) return rc;
    }
    const ve_estimator* e0 = b->members[0].get();
    const int W = cfg->window_size, F = W + 1;
    const size_t per_in = vb::ba_in_layout_max(W, e0->Lmax, e0->Mmax).total;  // one member's input block at full capacity
    // a batch rarely has every member at capacity: size the arenas for the full capacity of 8 members or a quarter of
    // the batch, whichever is larger (exhaustion is reported as VE_ERR_CAPACITY, never overrun)
    // per group: full capacity of 4 members or a quarter of the group, whichever is larger, plus a typical share for the rest
    size_t in_total = 0, out_total = 0;
    for (int g = 0; g < b->G; g++) {
        ve_batch::Group& grp = b->groups[g];
        const size_t at_cap = std::max<size_t>(std::min<size_t>(grp.count, 4), (size_t)(grp.count + 3) / 4);
        grp.in_base = in_total;
        grp.in_cap = per_in * at_cap;
        in_total += grp.in_cap;
        grp.out_base = out_total;
        grp.out_cap = vb::ba_out_reserve(F, e0->Lmax, true) * at_cap + vb::ba_out_reserve(F, 256, true) * (size_t)grp.count;
        out_total += grp.out_cap;
    }
    VB_CUDA_CHECK(b, VE_ERR_CUDA, b->d_seq.alloc(n));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, b->h_seq.alloc(n));
    std::memset(b->h_seq, 0, sizeof(vb::BaSeq) * n);
    VB_CUDA_CHECK(b, VE_ERR_CUDA, b->d_in.alloc(in_total));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, b->h_in.alloc(in_total));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, b->d_out.alloc(out_total));
    VB_CUDA_CHECK(b, VE_ERR_CUDA, b->h_out.alloc(out_total));
    b->w_in_global = vb::marg_w_in_global(vb::BA_MARG_MAX_DENSE, e0->nmax);
    b->pool.reset(new vb::HostPool(vb::HostPool::default_workers(n)));
    *out = b.release();
    return VE_OK;
}

void ve_batch_destroy(ve_batch* b) {
    vb::destroy_batch(b, [b] {
        for (int g = 0; b->groups && g < b->G; g++) {
            if (b->groups[g].stream) cudaStreamSynchronize(b->groups[g].stream);
            if (b->groups[g].copy_stream) cudaStreamSynchronize(b->groups[g].copy_stream);
        }
        b->pool.reset();
    });
}

int ve_batch_size(const ve_batch* b) { return vb::batch_size(b, VE_ERR_INVALID); }
int ve_batch_groups(const ve_batch* b) { return b ? b->G : VE_ERR_INVALID; }

ve_estimator* ve_batch_member(ve_batch* b, int k) { return vb::batch_member(b, k); }

const char* ve_batch_last_error(const ve_batch* b) { return vb::batch_last_error(b); }

int ve_batch_process_image(ve_batch* b, const int* active, const int* n, const int* const* ids, const double* const* xyz_uv_vel,
                           const double* stamps, int* status) {
    if (!b || !n || !ids || !xyz_uv_vel || !stamps) return VE_ERR_INVALID;
    std::vector<FrameMsg> msgs(b->S);
    for (int k = 0; k < b->S; k++) {
        msgs[k].active = active ? (active[k] != 0) : 1;
        msgs[k].n = n[k];
        msgs[k].ids = ids[k];
        msgs[k].obs = xyz_uv_vel[k];
        msgs[k].stamp = stamps[k];
        if (msgs[k].active && (n[k] < 0 || (n[k] && (!ids[k] || !xyz_uv_vel[k])))) return VE_ERR_INVALID;
    }
    return batch_process(b, msgs.data(), status);
}

int ve_batch_last_timing(const ve_batch* cb, float* ms4, int* launches) {
    if (!cb) return VE_ERR_INVALID;
    ve_batch* b = const_cast<ve_batch*>(cb);
    if (ms4) {
        if (b->marg_timing_valid) {
            cudaSetDevice(b->cfg.device);
            if (cudaEventSynchronize(b->groups[0].ev[3]) != cudaSuccess) return VE_ERR_CUDA;
            cudaEventElapsedTime(&b->last_ms[2], b->groups[0].ev[5], b->groups[0].ev[3]);
        }
        std::memcpy(ms4, b->last_ms, sizeof(b->last_ms));
    }
    if (launches) *launches = b->last_launches;
    return VE_OK;
}

int ve_batch_set_profile(ve_batch* b, int on) { return vb::set_profile(b, on, VE_ERR_INVALID, VE_ERR_CUDA); }

int ve_batch_kernel_times(const ve_batch* b, double* ms8, int* count8) { return vb::kernel_times(b, ms8, count8, 8, VE_ERR_INVALID); }

int ve_batch_sync(ve_batch* b) {
    if (!b) return VE_ERR_INVALID;
    VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaSetDevice(b->cfg.device));
    for (int g = 0; g < b->G; g++) VB_CUDA_CHECK(b, VE_ERR_CUDA, cudaStreamSynchronize(b->groups[g].stream));
    return VE_OK;
}

int ve_create(const ve_config* cfg, ve_estimator** out) { return vb::create_standalone(ve_batch_create, cfg, out, VE_ERR_INVALID); }

void ve_destroy(ve_estimator* e) { vb::destroy_standalone(e, ve_batch_destroy); }

const char* ve_last_error(const ve_estimator* e) { return vb::last_error(e); }

int ve_clear_state(ve_estimator* e) {
    if (!e) return VE_ERR_INVALID;
    clear_state(e);
    set_parameter(e);
    return VE_OK;
}

int ve_set_seed(ve_estimator* e, int n, const double* rows, const double* ba, const double* bg) {
    if (!e || n < 0 || (n && !rows) || !ba || !bg) return VE_ERR_INVALID;
    e->seeds.clear();
    for (int i = 0; i < n; i++) {
        const double* r = rows + 11 * i;
        SeedRow s;
        s.t = r[0];
        s.P = Vec3(r[1], r[2], r[3]);
        s.R = Quat(r[4], r[5], r[6], r[7]).normalized().R();
        s.V = Vec3(r[8], r[9], r[10]);
        e->seeds.push_back(s);
    }
    e->seed_ba = Vec3(ba[0], ba[1], ba[2]);
    e->seed_bg = Vec3(bg[0], bg[1], bg[2]);
    return VE_OK;
}

int ve_process_imu(ve_estimator* e, double dt, const double* acc, const double* gyr) {
    if (!e || !acc || !gyr) return VE_ERR_INVALID;
    process_imu(e, dt, Vec3(acc[0], acc[1], acc[2]), Vec3(gyr[0], gyr[1], gyr[2]));
    return VE_OK;
}

int ve_process_imu_batch(ve_estimator* e, int n, const double* dt, const double* acc, const double* gyr) {
    if (!e || n < 0 || (n && (!dt || !acc || !gyr))) return VE_ERR_INVALID;
    for (int i = 0; i < n; i++)
        process_imu(e, dt[i], Vec3(acc[3 * i], acc[3 * i + 1], acc[3 * i + 2]), Vec3(gyr[3 * i], gyr[3 * i + 1], gyr[3 * i + 2]));
    return VE_OK;
}

int ve_process_image(ve_estimator* e, int n, const int* ids, const double* xyz_uv_vel, double stamp) {
    if (!e || n < 0 || (n && (!ids || !xyz_uv_vel))) return VE_ERR_INVALID;
    if (const int rc = vb::refuse_member(e, VE_ERR_INVALID, "ve_process_image on a member of a batch: use ve_batch_process_image"))
        return rc;
    e->err.clear();
    FrameMsg m{1, n, ids, xyz_uv_vel, stamp};
    return batch_process(e->batch, &m, nullptr);
}

int ve_get_states(const ve_estimator* e, double* out, double* td) {
    if (!e || !out) return VE_ERR_INVALID;
    for (int i = 0; i <= e->W; i++) {
        double* o = out + 16 * i;
        const Quat q = Quat::FromR(e->Rs[i]);
        o[0] = e->Ps[i].x; o[1] = e->Ps[i].y; o[2] = e->Ps[i].z; o[3] = q.w; o[4] = q.x; o[5] = q.y; o[6] = q.z;
        o[7] = e->Vs[i].x; o[8] = e->Vs[i].y; o[9] = e->Vs[i].z;
        o[10] = e->Bas[i].x; o[11] = e->Bas[i].y; o[12] = e->Bas[i].z;
        o[13] = e->Bgs[i].x; o[14] = e->Bgs[i].y; o[15] = e->Bgs[i].z;
    }
    if (td) *td = e->td;
    return VE_OK;
}

int ve_set_relo_frame(ve_estimator* e, double frame_stamp, int frame_index, int n, const double* match_points, const double* relo_t,
                      const double* relo_r) {
    if (!e || n < 0 || (n && !match_points) || !relo_t || !relo_r) return VE_ERR_INVALID;
    e->relo_frame_stamp = frame_stamp;
    e->relo_frame_index = frame_index;
    e->match_points.assign(match_points, match_points + 3 * (size_t)n);
    e->prev_relo_t = Vec3(relo_t[0], relo_t[1], relo_t[2]);
    std::memcpy(e->prev_relo_r.m, relo_r, sizeof(e->prev_relo_r.m));
    int found = 0;
    for (int i = 0; i < e->W; i++)
        if (e->relo_frame_stamp == e->Headers[i]) {
            e->relo_frame_local_index = i;
            e->relocalization_info = true;
            for (int j = 0; j < 7; j++) e->relo_Pose[j] = e->para_Pose[i][j];
            found = 1;
        }
    return found;
}

int ve_get_features(const ve_estimator* e, int cap_features, int cap_obs, int* feature_id, int* start_frame, int* solve_flag,
                    double* estimated_depth, int* obs_offset, double* obs5) {
    if (!e) return VE_ERR_INVALID;
    int nf = (int)e->feature.size(), no = 0;
    for (auto& it : e->feature) no += (int)it.feature_per_frame.size();
    if (cap_features <= 0 && cap_obs <= 0) return nf;  // size query
    if (nf > cap_features || no > cap_obs || !obs_offset) return -nf - 1;
    int k = 0, o = 0;
    for (auto& it : e->feature) {
        if (feature_id) feature_id[k] = it.feature_id;
        if (start_frame) start_frame[k] = it.start_frame;
        if (solve_flag) solve_flag[k] = it.solve_flag;
        if (estimated_depth) estimated_depth[k] = it.estimated_depth;
        obs_offset[k] = o;
        for (auto& f : it.feature_per_frame) {
            if (obs5) {
                double* d = obs5 + 5 * (size_t)o;
                d[0] = f.point.x; d[1] = f.point.y; d[2] = f.point.z; d[3] = f.u; d[4] = f.v;
            }
            o++;
        }
        k++;
    }
    obs_offset[k] = o;
    return nf;
}

int ve_get_headers(const ve_estimator* e, double* stamps) {
    if (!e || !stamps) return VE_ERR_INVALID;
    for (int i = 0; i <= e->W; i++) stamps[i] = e->Headers[i];
    return VE_OK;
}

int ve_get_relocalization(const ve_estimator* e, double* o) {
    if (!e || !o) return VE_ERR_INVALID;
    std::memcpy(o, e->drift_correct_r.m, 9 * sizeof(double));
    o[9] = e->drift_correct_t.x; o[10] = e->drift_correct_t.y; o[11] = e->drift_correct_t.z;
    o[12] = e->relo_relative_t.x; o[13] = e->relo_relative_t.y; o[14] = e->relo_relative_t.z;
    o[15] = e->relo_relative_q.w; o[16] = e->relo_relative_q.x; o[17] = e->relo_relative_q.y; o[18] = e->relo_relative_q.z;
    o[19] = e->relo_relative_yaw;
    o[20] = e->relocalization_info ? 1.0 : 0.0;
    o[21] = e->relo_frame_local_index;
    o[22] = e->n_relo_factors;
    o[23] = e->n_relo_solves;
    return VE_OK;
}

int ve_debug_ex_rotation(int n_steps, const int* corres_off, const double* corres4, const double* dq_wxyz, int window_size, double* ric_out,
                         int* ok_out, double* cov_out, double* rc_out, const double* rc_in) {
    if (n_steps < 0 || !corres_off || !dq_wxyz || !ric_out || !ok_out) return VE_ERR_INVALID;
    vb::init::ExRotation cal;
    for (int k = 0; k < n_steps; k++) {
        std::vector<double> c(corres4 + 4 * (size_t)corres_off[k], corres4 + 4 * (size_t)corres_off[k + 1]);
        Mat3 out;
        const double* q = dq_wxyz + 4 * k;
        Mat3 given;
        if (rc_in) std::memcpy(given.m, rc_in + 9 * k, sizeof(given.m));
        ok_out[k] = cal.calibrate(c, Quat(q[0], q[1], q[2], q[3]), window_size, out, rc_in ? &given : nullptr) ? 1 : 0;
        std::memcpy(ric_out + 9 * k, cal.ric.m, 9 * sizeof(double));
        if (cov_out) cov_out[k] = cal.last_cov1;
        if (rc_out) std::memcpy(rc_out + 9 * k, cal.Rc.back().m, 9 * sizeof(double));
    }
    return VE_OK;
}

int ve_init_info(const ve_estimator* e, double* r) {
    if (!e) return VE_ERR_INVALID;
    if (r) {
        r[0] = e->init_l; r[1] = e->init_scale; r[2] = e->g.x; r[3] = e->g.y; r[4] = e->g.z;
        r[5] = e->init_iterations; r[6] = e->init_cost; r[7] = e->init_failures;
    }
    return e->self_initialised ? 1 : 0;
}

int ve_get_extrinsic(const ve_estimator* e, double* tic3, double* ric9) {
    if (!e) return VE_ERR_INVALID;
    if (tic3) { tic3[0] = e->tic.x; tic3[1] = e->tic.y; tic3[2] = e->tic.z; }
    if (ric9) std::memcpy(ric9, e->ric.m, 9 * sizeof(double));
    return VE_OK;
}

int ve_window_size(const ve_estimator* e) { return e ? e->W : VE_ERR_INVALID; }

int ve_get_latest_imu(const ve_estimator* e, double* acc0, double* gyr0, double* g3) {
    if (!e) return VE_ERR_INVALID;
    if (acc0) { acc0[0] = e->acc_0.x; acc0[1] = e->acc_0.y; acc0[2] = e->acc_0.z; }
    if (gyr0) { gyr0[0] = e->gyr_0.x; gyr0[1] = e->gyr_0.y; gyr0[2] = e->gyr_0.z; }
    if (g3) { g3[0] = e->g.x; g3[1] = e->g.y; g3[2] = e->g.z; }
    return VE_OK;
}

int ve_info(const ve_estimator* e, int* o, double* costs2) {
    if (!e || !o) return VE_ERR_INVALID;
    o[0] = e->solver_flag; o[1] = e->frame_count; o[2] = e->marginalization_flag; o[3] = e->n_solves; o[4] = e->n_reboots;
    o[5] = e->last_landmarks; o[6] = e->last_visual; o[7] = e->last_state.iteration; o[8] = e->last_state.successful;
    // termination coding: 0 iteration cap, 1 parameter tol, 2 function tol, 4 failure
    o[9] = e->last_state.done == 2 ? 1 : e->last_state.done == 3 ? 2 : e->last_state.done == 4 ? 4 : 0;
    if (costs2) {
        costs2[0] = e->last_state.initial_cost;
        costs2[1] = e->last_state.x_cost;
    }
    return VE_OK;
}

int ve_get_prior(const ve_estimator* ce, int cap, double* A, double* b, int* nblocks, int* blocks4) {
    if (!ce) return VE_ERR_INVALID;
    ve_estimator* e = const_cast<ve_estimator*>(ce);
    if (!e->has_prior || !e->marg_Araw) return 0;
    const int n = e->prior_n;
    if (n > cap) return -n;
    // the marginalisation that produced the prior may still be running: wait for the batch stream, then read the
    // un-floored Schur complement straight from device memory
    VB_CUDA_CHECK(e, VE_ERR_CUDA, cudaSetDevice(e->cfg.device));
    VB_CUDA_CHECK(e, VE_ERR_CUDA, cudaStreamSynchronize(e->batch->groups[e->member / e->batch->members_per_group].stream));
    VB_CUDA_CHECK(e, VE_ERR_CUDA, cudaMemcpy(A, e->marg_Araw, sizeof(double) * (size_t)n * n, cudaMemcpyDeviceToHost));
    VB_CUDA_CHECK(e, VE_ERR_CUDA, cudaMemcpy(b, e->marg_graw, sizeof(double) * n, cudaMemcpyDeviceToHost));
    if (nblocks) *nblocks = (int)e->prior_blocks.size();
    if (blocks4)
        for (size_t k = 0; k < e->prior_blocks.size(); k++) {
            blocks4[4 * k] = e->prior_blocks[k].type;
            blocks4[4 * k + 1] = e->prior_blocks[k].index;
            blocks4[4 * k + 2] = e->prior_blocks[k].off;
            blocks4[4 * k + 3] = e->prior_blocks[k].size;
        }
    return n;
}

int ve_set_profile(ve_estimator* e, int on) { return e ? ve_batch_set_profile(e->batch, on) : VE_ERR_INVALID; }

int ve_kernel_times(const ve_estimator* e, double* ms8, int* count8) { return e ? ve_batch_kernel_times(e->batch, ms8, count8) : VE_ERR_INVALID; }

int ve_last_traffic(const ve_estimator* e, double* h2d_bytes, double* d2h_bytes) {
    if (!e) return VE_ERR_INVALID;
    if (h2d_bytes) *h2d_bytes = (double)e->h2d_bytes;
    if (d2h_bytes) *d2h_bytes = (double)e->d2h_bytes;
    return VE_OK;
}

int ve_solver_debug(const ve_estimator* ce, double* out18) {
    if (!ce || !out18) return VE_ERR_INVALID;
    ve_estimator* e = const_cast<ve_estimator*>(ce);
    out18[0] = e->last_state.retries;
    out18[1] = e->last_state.mu;
    out18[2] = e->last_state.radius;
    for (int k = 0; k < 8; k++) out18[3 + k] = (double)e->last_state.clk[k];
    double sweeps[vb::BA_MARG_DIAG] = {};  // marg_solve_kernel's diagnostics behind the prior's n entries of graw
    if (e->has_prior && e->marg_graw) {
        VB_CUDA_CHECK(e, VE_ERR_CUDA, cudaSetDevice(e->cfg.device));
        VB_CUDA_CHECK(e, VE_ERR_CUDA, cudaStreamSynchronize(e->batch->groups[e->member / e->batch->members_per_group].stream));
        VB_CUDA_CHECK(e, VE_ERR_CUDA, cudaMemcpy(sweeps, e->marg_graw + e->marg_n, sizeof(sweeps), cudaMemcpyDeviceToHost));
    }
    out18[11] = sweeps[0];
    out18[12] = sweeps[1];
    for (int k = 0; k < 5; k++) out18[13 + k] = sweeps[2 + k];
    return VE_OK;
}

int ve_last_timing(const ve_estimator* e, float* ms4, int* launches) { return e ? ve_batch_last_timing(e->batch, ms4, launches) : VE_ERR_INVALID; }

// ---- single-factor test entries: the device code of the solve evaluated on caller-supplied blocks -------------------
int ve_debug_projection_factor(const double* params23, const double* data12, int use_td, double focal_length, double tr, double row,
                               int robust, double* out43) {
    if (!params23 || !data12 || !out43) return VE_ERR_INVALID;
    if (!vb::device_available(0)) return VE_ERR_NO_DEVICE;
    vb::DeviceArray<double> d;
    if (d.alloc(23 + 12 + 43) != cudaSuccess) return VE_ERR_CUDA;
    vb::BaDims dm{};
    dm.est_td = use_td ? 1 : 0;
    dm.sqrt_info_vis = focal_length / 1.5;
    dm.tr_over_row = tr / row;
    dm.half_row = row / 2;
    if (cudaMemcpy(d, params23, sizeof(double) * 23, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(d + 23, data12, sizeof(double) * 12, cudaMemcpyHostToDevice) != cudaSuccess)
        return VE_ERR_CUDA;
    vb::launch_debug_visual(dm, d, d + 23, robust, d + 35, nullptr);
    return cudaMemcpy(out43, d + 35, sizeof(double) * 43, cudaMemcpyDeviceToHost) == cudaSuccess ? VE_OK : VE_ERR_CUDA;
}

int ve_debug_imu_factor(const double* noise4, double g_norm, const double* ba, const double* bg, int n, const double* dt,
                        const double* acc, const double* gyr, const double* params32, double* out_preint, double* out_factor) {
    if (!noise4 || !ba || !bg || n < 1 || !dt || !acc || !gyr) return VE_ERR_INVALID;
    if (!vb::device_available(0)) return VE_ERR_NO_DEVICE;
    // sample 0 seeds the IntegrationBase (acc_0 / gyr_0), samples 1..n-1 are pushed with dt[k]
    vb::BaSeq q{};
    vb::PreintJob jobs[2]{};
    jobs[0].type = 0;
    for (int c = 0; c < 3; c++) {
        jobs[0].acc0[c] = acc[c];
        jobs[0].gyr0[c] = gyr[c];
        jobs[0].ba[c] = ba[c];
        jobs[0].bg[c] = bg[c];
    }
    jobs[1].type = 1;
    jobs[1].n = n - 1;
    std::vector<double> rec(7 * (size_t)std::max(n - 1, 1));
    for (int k = 1; k < n; k++) {
        double* r = &rec[7 * (size_t)(k - 1)];
        r[0] = dt[k];
        for (int c = 0; c < 3; c++) {
            r[1 + c] = acc[3 * k + c];
            r[4 + c] = gyr[3 * k + c];
        }
    }
    vb::DeviceArray<unsigned char> d;
    using vb::ba_align16;
    const size_t o_seq = 0, o_jobs = ba_align16(sizeof(vb::BaSeq)), o_rec = o_jobs + ba_align16(sizeof(jobs)),
                 o_pre = o_rec + ba_align16(rec.size() * sizeof(double)), o_prm = o_pre + ba_align16(sizeof(vb::PreInt)),
                 o_out = o_prm + ba_align16(32 * sizeof(double)), total = o_out + ba_align16(465 * sizeof(double));
    if (d.alloc(total) != cudaSuccess) return VE_ERR_CUDA;
    q.n_jobs = 2;
    q.sqrt_mask = 1u;
    q.jobs = reinterpret_cast<const vb::PreintJob*>(d + o_jobs);
    q.samples = reinterpret_cast<const double*>(d + o_rec);
    for (int c = 0; c < 4; c++) q.noise[c] = noise4[c];
    q.p.preint = reinterpret_cast<vb::PreInt*>(d + o_pre);
    vb::BaDims dm{};
    dm.G[2] = g_norm;
    if (cudaMemcpy(d + o_seq, &q, sizeof(q), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(d + o_jobs, jobs, sizeof(jobs), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(d + o_rec, rec.data(), rec.size() * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
        (params32 && cudaMemcpy(d + o_prm, params32, 32 * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess))
        return VE_ERR_CUDA;
    vb::BatchShape sh{};
    sh.S = 1;
    sh.W = 0;
    sh.any_jobs = 1;
    vb::launch_preint_jobs(reinterpret_cast<vb::BaSeq*>(d + o_seq), sh, nullptr, nullptr, nullptr);
    if (params32 && out_factor) {
        vb::launch_debug_imu(dm, reinterpret_cast<const vb::PreInt*>(d + o_pre), reinterpret_cast<const double*>(d + o_prm),
                             reinterpret_cast<double*>(d + o_out), nullptr);
        if (cudaMemcpy(out_factor, d + o_out, 465 * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) return VE_ERR_CUDA;
    }
    if (out_preint) {
        vb::PreInt pre;
        if (cudaMemcpy(&pre, d + o_pre, sizeof(pre), cudaMemcpyDeviceToHost) != cudaSuccess) return VE_ERR_CUDA;
        // sum_dt | dp 3 | dq 4 (wxyz) | dv 3 | jac 225 | cov 225 | sqrt_info 225
        out_preint[0] = pre.sum_dt;
        std::memcpy(out_preint + 1, pre.dp, 3 * sizeof(double));
        std::memcpy(out_preint + 4, pre.dq, 4 * sizeof(double));
        std::memcpy(out_preint + 8, pre.dv, 3 * sizeof(double));
        std::memcpy(out_preint + 11, pre.jac, 225 * sizeof(double));
        std::memcpy(out_preint + 236, pre.cov, 225 * sizeof(double));
        std::memcpy(out_preint + 461, pre.sqrt_info, 225 * sizeof(double));
    }
    return cudaGetLastError() == cudaSuccess ? VE_OK : VE_ERR_CUDA;
}

}  // extern "C"
