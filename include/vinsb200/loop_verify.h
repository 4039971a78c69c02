/* vinsb200 loop verification — C ABI of the geometric check of a loop candidate (KeyFrame::findConnection,
 * pose_graph/src/keyframe.cpp:259-520), on the device, for the graphs of pose_graph.h.
 *
 * Which old key frame is the candidate stays with the caller (place recognition, a GPS prior, ground truth); this API
 * decides whether the pair is a loop and, when it is, returns the loop measurement vp_add_keyframe / vp_update_loop take
 * and the matched points ve_set_relo_frame takes.
 *
 *   vp_loop_enable / vp_batch_loop_enable   allocate the descriptor arena: one slot per key frame index (0 ..
 *                            max_keyframes - 1) of every member, resident in device memory.  The BRIEF pattern (256
 *                            pairs x1 y1 x2 y2, support_files/brief_pattern.yml) is copied at this call.  PINHOLE;
 *                            vp_loop_enable_camera (loop_camera.h) takes MEI and KANNALA_BRANDT cameras.
 *                            Per slot about 12 + 32 + 28 bytes per window point and 48 bytes per corner.
 *   vp_attach_keyframe       the KeyFrame constructor's computeWindowBRIEFPoint + computeBRIEFPoint (:75-113): the image
 *                            (rows x cols, 8-bit), the key frame's VIO pose as created (origin_vio_T / origin_vio_R) and its
 *                            n window points (point_3d, point_2d_uv, point_2d_norm, point_id).  GaussianBlur 9x9 sigma 2,
 *                            FAST-9 (threshold 20, non-max suppression), BRIEF on both point sets and liftProjective of the
 *                            corners run on the device; the call returns once the slot is written.  n > max_window or more
 *                            corners than max_corners is VP_ERR_CAPACITY and leaves the slot as it was.
 *   vp_find_connection       findConnection(old) for two attached slots: Hamming matching (best < 80, the first index of the
 *                            smallest distance), more than 25 matches, PnP-RANSAC (float64, see DESIGN §5: not OpenCV's
 *                            sampler or solver), more than 25 inliers, |relative_yaw| < 30 and |relative_t| < 20.
 *                            match_xyid (cap x 3, may be NULL) = the inliers' (old normalised x, y, feature id) in window
 *                            order: ve_set_relo_frame's match_points.
 *   vp_batch_find_connection one launch chain for every member k with cur[k] >= 0 (results r[k], lists at
 *                            match_xyid + 3 cap k); status[k] (may be NULL) 1 = verified, 0 = skipped, < 0 error.
 *   vp_loop_last_timing      device ms (CUDA events) of the last attach (blur, FAST, BRIEF) and of the last verification
 *                            launch chain (matching, hypotheses, refit).
 *
 * A key frame loaded by vp_load (pose_graph.h) has a slot with its saved corners and descriptors and no window points:
 * it can be `old` of vp_find_connection; as `cur` it matches nothing.
 *
 * Errors return < 0 and change neither the graph nor any slot.  The vp_debug_* entries run one stage each on device 0
 * with no handle.
 */
#ifndef VINSB200_LOOP_VERIFY_H
#define VINSB200_LOOP_VERIFY_H

#include <stddef.h>
#include <stdint.h>

#include "pose_graph.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vp_loop_config {
    int rows, cols;            /* image size (ROW, COL): 8 .. 1024 rows, 8 .. 2048 columns */
    double intrinsics[8];      /* PINHOLE: fx fy cx cy k1 k2 p1 p2 (other models: loop_camera.h) */
    double ric9[9];            /* camera-to-body rotation qic, row-major */
    double tic3[3];            /* camera-to-body translation tic */
    const int* brief_pattern;  /* 256 x (x1, y1, x2, y2) */
    int max_window;            /* window points per key frame: 1 .. 1024 */
    int max_corners;           /* FAST corners per key frame: 1 .. 65536 */
} vp_loop_config;

typedef struct vp_loop_result {
    int accepted;         /* 1: the pair is a loop */
    int n_matches;        /* window points with a BRIEF match */
    int n_inliers;        /* PnP consensus set (0 when PnP did not run) */
    int n_points;         /* rows written to match_xyid */
    double loop_info[8];  /* relative t (3), relative q (w x y z), relative yaw (degrees) */
    double old_R9[9];     /* PnP_R_old, row-major: the old key frame's body pose in the current VIO frame */
    double old_T3[3];     /* PnP_T_old */
} vp_loop_result;

int vp_loop_enable(vp_graph* g, const vp_loop_config* cfg);
int vp_batch_loop_enable(vp_batch* b, const vp_loop_config* cfg);
int vp_attach_keyframe(vp_graph* g, int index, const double* vio_P3, const double* vio_Qwxyz, const uint8_t* img, size_t row_stride,
                       int n, const float* point_3d, const float* point_uv, const float* point_norm, const double* point_id,
                       int* n_corners);
int vp_find_connection(vp_graph* g, int cur, int old, vp_loop_result* r, int cap, double* match_xyid);
int vp_batch_find_connection(vp_batch* b, const int* cur, const int* old, vp_loop_result* r, int cap, double* match_xyid, int* status);
/* ms6 = blur, FAST (with the corner lift), BRIEF (last attach) | matching, hypotheses, refit (last verification) */
int vp_loop_last_timing(vp_graph* g, float* ms6);
int vp_batch_loop_last_timing(vp_batch* b, float* ms6);

/* ---- one stage each, device 0, no handle (images rows x cols, dense) */
int vp_debug_brief_blur(const uint8_t* img, int rows, int cols, uint8_t* out);
/* FAST corners (x, y) in row-major order; returns the count, VP_ERR_CAPACITY above cap */
int vp_debug_fast(const uint8_t* img, int rows, int cols, int cap, float* xy);
/* BRIEF of n (<= 1024) points: desc n x 4 words */
int vp_debug_brief(const uint8_t* img, int rows, int cols, const int* pattern, int n, const float* uv, uint64_t* desc);
/* searchByBRIEFDes of na (<= 1024) descriptors against nb: idx[i] = matched index or -1 */
int vp_debug_match(int na, const uint64_t* a, int nb, const uint64_t* b, int* idx);
/* PnP-RANSAC of n (26 .. 1024) correspondences: Rt12 = R (row-major) | t, world to camera; inlier (may be NULL) = mask */
int vp_debug_pnp(int n, const float* point_3d, const float* norm, double* Rt12, int* n_inliers, uint8_t* inlier);

#ifdef __cplusplus
}
#endif
#endif
