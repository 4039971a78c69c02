/* vinsb200 loop verification for every camera model of the tracker — the part of the loop_verify.h C ABI that names the
 * camera.  In the reference the camera enters findConnection in one place: computeBRIEFPoint lifts each FAST corner with
 * m_camera->liftProjective and divides by z (pose_graph/src/keyframe.cpp:108), with m_camera read from the same YAML file
 * as the tracker's camera.  Blur, FAST, BRIEF, matching, PnP with K = I and the loop gate do not depend on it.
 *
 *   vp_loop_enable_camera / vp_batch_loop_enable_camera   vp_loop_enable / vp_batch_loop_enable with the camera model;
 *                    cfg->intrinsics is read in vt_config's order for that model:
 *                      VP_CAMERA_PINHOLE          fx fy cx cy k1 k2 p1 p2
 *                      VP_CAMERA_MEI              gamma1 gamma2 u0 v0 k1 k2 p1 p2, plus xi (mirror_parameters.xi)
 *                      VP_CAMERA_KANNALA_BRANDT   mu mv u0 v0 k2 k3 k4 k5
 *                    xi is ignored by the other two models.  A model out of range, a non-finite xi or any configuration
 *                    error of vp_loop_enable is VP_ERR_INVALID, and nothing is allocated.  vp_loop_enable(g, cfg) is
 *                    vp_loop_enable_camera(g, cfg, VP_CAMERA_PINHOLE, 0).
 *   vp_debug_lift    the device lift of the corners (liftProjective / z) for n float pixel positions uv (n x 2), on device 0
 *                    with no handle; xy (n x 2) is stored as float, exactly as in a key-frame slot.  n = 1 .. 65536.
 */
#ifndef VINSB200_LOOP_CAMERA_H
#define VINSB200_LOOP_CAMERA_H

#include "loop_verify.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the values of vt_camera_model (tracker.h) */
typedef enum vp_camera_model { VP_CAMERA_PINHOLE = 0, VP_CAMERA_MEI = 1, VP_CAMERA_KANNALA_BRANDT = 2 } vp_camera_model;

int vp_loop_enable_camera(vp_graph* g, const vp_loop_config* cfg, int camera_model, double xi);
int vp_batch_loop_enable_camera(vp_batch* b, const vp_loop_config* cfg, int camera_model, double xi);
int vp_debug_lift(int camera_model, const double* intrinsics8, double xi, int n, const float* uv, float* xy);

#ifdef __cplusplus
}
#endif
#endif
