// Handle-free C entries of the initialisation stages (include/vinsb200/estimator.h, "Initialisation"): plain arrays in,
// plain arrays out, no device needed.
#include <cstring>

#include "initial.h"
#include "vinsb200/estimator.h"

using namespace vb::init;
using vb::Mat3;
using vb::Quat;
using vb::Vec3;

namespace {
std::vector<Track> make_tracks(int n, const int* ids, const int* start, const int* nobs, const double* xy) {
    std::vector<Track> t(n);
    size_t off = 0;
    for (int i = 0; i < n; i++) {
        t[i].id = ids[i];
        t[i].start_frame = start[i];
        t[i].xy.assign(xy + 2 * off, xy + 2 * (off + nobs[i]));
        off += nobs[i];
    }
    return t;
}
}  // namespace

extern "C" {

int ve_debug_relative_rt(const double* corres4, int n, double* R9, double* T3, int* inliers) {
    if (!corres4 || n < 0 || !R9 || !T3) return VE_ERR_INVALID;
    Mat3 R;
    Vec3 T;
    int cnt = 0;
    const bool ok = solve_relative_rt(std::vector<double>(corres4, corres4 + 4 * (size_t)n), R, T, &cnt);
    std::memcpy(R9, R.m, sizeof(R.m));
    T3[0] = T.x; T3[1] = T.y; T3[2] = T.z;
    if (inliers) *inliers = cnt;
    return ok ? 1 : 0;
}

int ve_debug_solve_pnp(const double* pts3, const double* pts2, int n, double* R9, double* t3) {
    if (!pts3 || !pts2 || n < 0 || !R9 || !t3) return VE_ERR_INVALID;
    Mat3 R;
    std::memcpy(R.m, R9, sizeof(R.m));
    Vec3 t(t3[0], t3[1], t3[2]);
    const bool ok = solve_pnp(std::vector<double>(pts3, pts3 + 3 * (size_t)n), std::vector<double>(pts2, pts2 + 2 * (size_t)n), R, t);
    std::memcpy(R9, R.m, sizeof(R.m));
    t3[0] = t.x; t3[1] = t.y; t3[2] = t.z;
    return ok ? 1 : 0;
}

int ve_debug_sfm_construct(int frame_num, int l, const double* relative_R9, const double* relative_T3, int n_tracks,
                           const int* track_ids, const int* track_start, const int* track_nobs, const double* track_xy,
                           double function_tolerance, double* q_wxyz, double* T, int* n_pts, int* pt_ids, double* pts, int* iterations,
                           double* final_cost) {
    if (frame_num < 2 || l < 0 || l >= frame_num - 1 || !relative_R9 || !relative_T3 || n_tracks < 0 || !q_wxyz || !T) return VE_ERR_INVALID;
    Mat3 R;
    std::memcpy(R.m, relative_R9, sizeof(R.m));
    const Vec3 t(relative_T3[0], relative_T3[1], relative_T3[2]);
    std::vector<Quat> q;
    std::vector<Vec3> Tv;
    std::map<int, Vec3> tracked;
    const bool ok = sfm_construct(frame_num, q, Tv, l, R, t, make_tracks(n_tracks, track_ids, track_start, track_nobs, track_xy), tracked,
                                  iterations, final_cost, function_tolerance > 0 ? function_tolerance : 1e-6);
    for (int i = 0; i < frame_num; i++) {
        q_wxyz[4 * i] = q[i].w; q_wxyz[4 * i + 1] = q[i].x; q_wxyz[4 * i + 2] = q[i].y; q_wxyz[4 * i + 3] = q[i].z;
        T[3 * i] = Tv[i].x; T[3 * i + 1] = Tv[i].y; T[3 * i + 2] = Tv[i].z;
    }
    int k = 0;
    for (auto& kv : tracked) {
        if (pt_ids) pt_ids[k] = kv.first;
        if (pts) { pts[3 * k] = kv.second.x; pts[3 * k + 1] = kv.second.y; pts[3 * k + 2] = kv.second.z; }
        k++;
    }
    if (n_pts) *n_pts = k;
    return ok ? 1 : 0;
}

int ve_debug_initial_structure(int F, const double* headers, int n_all, const double* stamps, const int* pts_off,
                               const int* pt_ids, const double* pt_xy, const int* imu_off, const double* imu7,
                               const double* lin6, int n_tracks, const int* track_ids, const int* track_start,
                               const int* track_nobs, const double* track_xy, const double* ric9, const double* tic3,
                               double g_norm, double function_tolerance, double* frame_R, double* frame_T, double* x, double* g3,
                               double* delta_bg3, int* info4, double* bundle_cost) {
    if (F < 3 || n_all < F || !headers || !stamps || !pts_off || !imu_off || !ric9 || !tic3) return VE_ERR_INVALID;
    std::vector<ImageFrame> frames(n_all);
    for (int k = 0; k < n_all; k++) {
        ImageFrame& fr = frames[k];
        fr.t = stamps[k];
        fr.ids.assign(pt_ids + pts_off[k], pt_ids + pts_off[k + 1]);
        fr.xy.assign(pt_xy + 2 * (size_t)pts_off[k], pt_xy + 2 * (size_t)pts_off[k + 1]);
        if (k > 0) {
            const double* l = lin6 + 6 * k;
            fr.pre.start(Vec3(l[0], l[1], l[2]), Vec3(l[3], l[4], l[5]), Vec3(), Vec3());
            for (int s = imu_off[k]; s < imu_off[k + 1]; s++) {
                const double* r = imu7 + 7 * (size_t)s;
                fr.pre.push_back(r[0], Vec3(r[1], r[2], r[3]), Vec3(r[4], r[5], r[6]));
            }
        }
    }
    Mat3 ric;
    std::memcpy(ric.m, ric9, sizeof(ric.m));
    std::vector<Vec3> Bgs(F);
    std::vector<double> xv;
    const Result res = initial_structure(frames, std::vector<double>(headers, headers + F),
                                         make_tracks(n_tracks, track_ids, track_start, track_nobs, track_xy), ric,
                                         Vec3(tic3[0], tic3[1], tic3[2]), g_norm, Bgs, xv,
                                         function_tolerance > 0 ? function_tolerance : 1e-6);
    int keys = 0;
    for (int k = 0; k < n_all; k++) {
        if (frame_R) std::memcpy(frame_R + 9 * k, frames[k].R.m, 9 * sizeof(double));
        if (frame_T) { frame_T[3 * k] = frames[k].T.x; frame_T[3 * k + 1] = frames[k].T.y; frame_T[3 * k + 2] = frames[k].T.z; }
        keys += frames[k].is_key_frame;
    }
    if (x && res.code == 0) std::memcpy(x, xv.data(), sizeof(double) * xv.size());
    if (g3) { g3[0] = res.g.x; g3[1] = res.g.y; g3[2] = res.g.z; }
    if (delta_bg3) { delta_bg3[0] = res.delta_bg.x; delta_bg3[1] = res.delta_bg.y; delta_bg3[2] = res.delta_bg.z; }
    if (info4) { info4[0] = res.l; info4[1] = res.sfm_iterations; info4[2] = keys; info4[3] = 0; }
    if (bundle_cost) *bundle_cost = res.sfm_cost;
    return res.code;
}

}  // extern "C"
