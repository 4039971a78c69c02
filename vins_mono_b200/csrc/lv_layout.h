// Layouts of the loop-verification buffers (lv_kernels.cu, loop_verify.cpp): the key-frame descriptor arena (one slot
// per key frame of each graph, resident in device memory), the staging block of one key-frame attach, its scratch, and
// the per-verification scratch and result block.  Each layout is defined here once; host and device code share it and
// tests/hostlib/lv_layout_host.cpp checks it with g++.
#pragma once
#include <cstddef>
#include <cstdint>

#ifdef __CUDACC__
#define LV_LAYOUT_FN __host__ __device__ constexpr inline
#else
#define LV_LAYOUT_FN constexpr inline
#endif

namespace vb {

// keyframe.cpp / BRIEF.cpp constants
constexpr int LV_BITS = 256, LV_WORDS = 4;       // 256-bit BRIEF, 4 x 64-bit words, bit i in word i / 64
constexpr int LV_FAST_THRESHOLD = 20;            // computeBRIEFPoint's fast_th
constexpr int LV_MATCH_INIT = 128, LV_MATCH_ACCEPT = 80;  // searchInAera: bestDist starts at 128, accepted below 80
constexpr int LV_MIN_LOOP_NUM = 25;              // keyframe.h MIN_LOOP_NUM: more than this many matches / inliers
// PnP-RANSAC: hypotheses scored in parallel (one warp each), each from LV_SAMPLE correspondences (6-point DLT)
constexpr int LV_HYP = 128, LV_SAMPLE = 6;
constexpr double LV_PNP_THRESHOLD = 10.0 / 460.0;  // PnPRANSAC's reprojection threshold in normalised coordinates
constexpr int LV_REFIT_ITERS = 10;
// capacities accepted by vp_loop_enable
constexpr int LV_CAP_WINDOW = 1024, LV_CAP_CORNERS = 65536, LV_MAX_ROWS = 1024, LV_MAX_COLS = 2048;

LV_LAYOUT_FN size_t lv_align16(size_t b) { return (b + 15) & ~(size_t)15; }

// ---- header of a key-frame slot and of an attach staging block
struct LvSlotHdr {
    double vio_P[3], vio_Q[4];  // the key frame's VIO pose as it was created (origin_vio_T / origin_vio_R)
    int n_win, n_corners, attached, pad;
};

// ---- a key-frame slot of the descriptor arena, in bytes, every array 16-byte aligned:
//      header | window 3-D points (float x 3) | window uv (float x 2) | window normalised (float x 2) | window ids (double) |
//      window descriptors (4 x u64) | corners (float x 2, pixel) | corners normalised (float x 2) | corner descriptors
struct LvSlotLayout {
    size_t hdr, p3d, uv, norm, id, wdesc, kp, kpn, kdesc, total;
};
LV_LAYOUT_FN LvSlotLayout lv_slot_layout(int max_window, int max_corners) {
    const size_t w = (size_t)max_window, c = (size_t)max_corners;
    LvSlotLayout o{0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    o.p3d = lv_align16(sizeof(LvSlotHdr));
    o.uv = o.p3d + lv_align16(12 * w);
    o.norm = o.uv + lv_align16(8 * w);
    o.id = o.norm + lv_align16(8 * w);
    o.wdesc = o.id + lv_align16(8 * w);
    o.kp = o.wdesc + lv_align16(32 * w);
    o.kpn = o.kp + lv_align16(8 * c);
    o.kdesc = o.kpn + lv_align16(8 * c);
    o.total = o.kdesc + lv_align16(32 * c);
    return o;
}
// bytes of the arena: S graphs x cap_kf slots
LV_LAYOUT_FN size_t lv_arena_bytes(int S, int cap_kf, int max_window, int max_corners) {
    return (size_t)S * (size_t)cap_kf * lv_slot_layout(max_window, max_corners).total;
}

// ---- staging block of one attach (host-to-device copy), in bytes: header | image rows x cols | window arrays as in
//      the slot
struct LvStageLayout {
    size_t hdr, img, p3d, uv, norm, id, total;
};
LV_LAYOUT_FN LvStageLayout lv_stage_layout(int rows, int cols, int max_window) {
    const size_t w = (size_t)max_window;
    LvStageLayout o{0, 0, 0, 0, 0, 0, 0};
    o.img = lv_align16(sizeof(LvSlotHdr));
    o.p3d = o.img + lv_align16((size_t)rows * cols);
    o.uv = o.p3d + lv_align16(12 * w);
    o.norm = o.uv + lv_align16(8 * w);
    o.id = o.norm + lv_align16(8 * w);
    o.total = o.id + lv_align16(8 * w);
    return o;
}
// the packed stage of one attach call (one host-to-device copy): per job its slot's byte offset in the arena (long long),
// padded to 16 bytes | per job a staging block at lv_stage_layout's total stride
LV_LAYOUT_FN size_t lv_attach_jobs_bytes(int n_jobs) { return lv_align16(8 * (size_t)n_jobs); }

// ---- staging of the key frames one vp_load puts into their slots (one host-to-device copy), in bytes: per key frame a
//      job (slot byte offset in the arena, block byte offset in the staging buffer: 2 x long long) | per key frame a
//      block of n corners: header (n_win 0) | corners (float x 2) | corners normalised (float x 2) | descriptors
struct LvLoadLayout {
    size_t hdr, kp, kpn, kdesc, total;
};
LV_LAYOUT_FN size_t lv_load_jobs_bytes(int n_kf) { return lv_align16(16 * (size_t)n_kf); }
LV_LAYOUT_FN LvLoadLayout lv_load_layout(int n) {
    const size_t c = (size_t)n;
    LvLoadLayout o{0, 0, 0, 0, 0};
    o.kp = lv_align16(sizeof(LvSlotHdr));
    o.kpn = o.kp + lv_align16(8 * c);
    o.kdesc = o.kpn + lv_align16(8 * c);
    o.total = o.kdesc + lv_align16(32 * c);
    return o;
}

// ---- scratch of one attach, in bytes: blurred image | FAST score map | survivor map | survivors per row |
//      status (corner count, overflow)
struct LvAttachLayout {
    size_t blur, score, keep, rowcnt, status, total;
};
LV_LAYOUT_FN LvAttachLayout lv_attach_layout(int rows, int cols) {
    const size_t px = (size_t)rows * cols;
    LvAttachLayout o{0, 0, 0, 0, 0, 0};
    o.score = lv_align16(px);
    o.keep = o.score + lv_align16(px);
    o.rowcnt = o.keep + lv_align16(px);
    o.status = o.rowcnt + lv_align16(4 * (size_t)rows);
    o.total = o.status + 16;
    return o;
}

// ---- scratch of one verification, in bytes: the cur / old slot indices and match count (4 ints) | per window point its
//      old corner (-1) | matched window indices in window order | per hypothesis its consensus count | its pose
//      (R row-major, t: world to old camera)
struct LvConnLayout {
    size_t hdr, win_match, midx, hyp_cnt, hyp_pose, total;
};
LV_LAYOUT_FN LvConnLayout lv_conn_layout(int max_window) {
    const size_t w = (size_t)max_window;
    LvConnLayout o{0, 0, 0, 0, 0, 0};
    o.win_match = 16;
    o.midx = o.win_match + lv_align16(4 * w);
    o.hyp_cnt = o.midx + lv_align16(4 * w);
    o.hyp_pose = o.hyp_cnt + lv_align16(4 * (size_t)LV_HYP);
    o.total = o.hyp_pose + lv_align16(8 * 12 * (size_t)LV_HYP);
    return o;
}

// ---- result block of one verification, in doubles:
//      accepted, matches, inliers, points written, best hypothesis, 3 spare | loop_info 8 (t, q wxyz, yaw degrees) |
//      PnP_R_old 9 | PnP_T_old 3 | R_old^T R_cur 9 (row-major; the host turns it into loop_info's q) | 3 spare |
//      inlier list max_window x (old normalised x, y, feature id)
constexpr int LV_RES_LOOP = 8, LV_RES_R = 16, LV_RES_T = 25, LV_RES_RQ = 28, LV_RES_LIST = 40;
LV_LAYOUT_FN size_t lv_result_doubles(int max_window) { return (size_t)LV_RES_LIST + 3 * (size_t)max_window; }

}  // namespace vb
