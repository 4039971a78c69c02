/* vinsb200 batched key-frame attach — the part of the loop_verify.h C ABI that attaches many key frames, of any members
 * of a batch, in one launch chain.  Each job is what vp_attach_keyframe does for one key frame (the KeyFrame
 * constructor's computeWindowBRIEFPoint + computeBRIEFPoint, pose_graph/src/keyframe.cpp:75-113), and the results are the
 * same bit for bit; vp_attach_keyframe itself is a one-job call of this path.  A replay of many sequences, where almost
 * every step makes a key frame in every member, attaches a step's key frames together instead of one after another.
 *
 *   vp_batch_attach_keyframes   n_jobs attaches in one launch chain: one host-to-device copy of the packed host images and
 *                    window arrays, one device-to-device 2-D copy per device image (img_on_device), the six attach kernels
 *                    over every job (gridDim.z = n_jobs), one copy of the per-job status back, one wait.  Jobs may name
 *                    several members and several slots of one member.
 *                    n_corners[j] (may be NULL) = job j's corner count.  status[j] (may be NULL) = 0, or VP_ERR_CAPACITY
 *                    when job j's corners exceed max_corners: that slot stays as it was, the other jobs are written, and
 *                    the call returns VP_ERR_CAPACITY.
 *                    A bad member or index, a null pointer, row_stride < cols, n outside 0 .. max_window or the same
 *                    (member, index) twice is VP_ERR_INVALID before anything runs, with status[j] = VP_ERR_INVALID for the
 *                    first such job; no slot changes.  More than 65535 jobs is VP_ERR_CAPACITY.  The staging buffers grow
 *                    to the largest call (about rows x cols bytes of stage and 3 rows x cols of scratch per job); an
 *                    allocation that fails is VP_ERR_CAPACITY and changes nothing.
 *                    vp_batch_loop_last_timing reports the call's blur, FAST and BRIEF stages over all its jobs.
 *                    A device image must be complete when the call is made: it is copied on the batch's own stream, which
 *                    does not wait for work on other streams, so the caller first synchronises the stream (or waits for
 *                    the event) that wrote it.  The call returns once its copies are done; the image may be reused then.
 */
#ifndef VINSB200_LOOP_ATTACH_H
#define VINSB200_LOOP_ATTACH_H

#include "loop_verify.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One key frame: vp_attach_keyframe's arguments plus the member (0 .. size - 1) and where the image lives
 * (img_on_device = 1: img is device memory on the batch's device, rows x cols at row_stride bytes). */
typedef struct vp_attach_job {
    int member, index;
    const double *vio_P3, *vio_Qwxyz;
    const uint8_t* img;
    size_t row_stride;
    int img_on_device;
    int n;
    const float *point_3d, *point_uv, *point_norm;
    const double* point_id;
} vp_attach_job;

int vp_batch_attach_keyframes(vp_batch* b, int n_jobs, const vp_attach_job* jobs, int* n_corners, int* status);

#ifdef __cplusplus
}
#endif
#endif
