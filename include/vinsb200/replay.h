/* vinsb200 replay driver — C ABI of the two node loops around the hot path, for offline sequences.
 *
 * Restates, for data already in memory instead of ROS topics:
 *   feature_tracker_node.cpp:28-165  img_callback: every image goes through vt_node_image (first-frame / discontinuity /
 *                                    frequency gating, readImage, updateID), a feature message is produced when it
 *                                    publishes (track_cnt > 1 points; x, y, z = 1 and the id/u/v/velocity channels
 *                                    travel as float32 exactly like sensor_msgs/PointCloud)
 *   estimator_node.cpp:98-136        getMeasurements: the IMU samples up to the image stamp plus the first one after it
 *   estimator_node.cpp:167-172       feature_callback drops the very first feature message
 *   estimator_node.cpp:225-265       process(): per-sample dt, linear interpolation of the sample that straddles the stamp
 *   estimator_node.cpp:275-316       image map construction and Estimator::processImage
 * The reference runs the two loops in two processes.  Here a session is a list of lanes.  A lane is a contiguous run of
 * sequences with one tracker thread and one estimator thread, coupled by a bounded queue (depth 2); all lanes run
 * concurrently on one GPU (each handle owns its CUDA stream).  vr_open makes a lane per sequence, vr_open_batch one lane
 * of all its sequences.  Both run the same two loops, which differ only in the library call of a step: a lane of one
 * calls its sequence's own handles, a batch lane steps all its sequences with one batch call.  No ROS, no CPU fallback:
 * the handles are the CUDA ones of tracker.h / estimator.h.
 */
#ifndef VINSB200_REPLAY_H
#define VINSB200_REPLAY_H

#include <stddef.h>
#include <stdint.h>

#include "vinsb200/estimator.h"
#include "vinsb200/tracker.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vr_sequence {
    const uint8_t* images;  /* n_images frames, frame k at images + k * frame_stride (host or device memory) */
    size_t row_stride, frame_stride;
    int n_images;
    int images_on_device;   /* 0: host pointers (each frame is copied to the GPU inside the call), 1: device pointers */
    const double* stamps;   /* n_images image time stamps (s) */
    int n_imu;
    const double* imu_t;    /* n_imu sample stamps (s), ascending */
    const double* acc;      /* n_imu x 3 linear_acceleration */
    const double* gyr;      /* n_imu x 3 angular_velocity */
} vr_sequence;

typedef struct vr_session vr_session;

/* The session borrows the handles and the sequence memory: they must outlive it.  Seed / configure the estimators
 * before the first vr_advance. */
int vr_open(int n_seq, vt_tracker* const* trackers, ve_estimator* const* estimators, const vr_sequence* seqs, vr_session** out);
/* Batch mode: the sequences are the members of one tracker batch and one estimator batch (same count, same order; all
 * sequences with the same row_stride and images_on_device).  The session is then ONE lane: every image step is a
 * vt_batch_node_image call, every published step a ve_batch_process_image call (one launch chain for all sequences);
 * vr_stats reports the batch's kernel launches on sequence 0. */
int vr_open_batch(vt_batch* trackers, ve_batch* estimators, const vr_sequence* seqs, vr_session** out);
void vr_close(vr_session* s);
const char* vr_last_error(const vr_session* s);

/* Runs every sequence forward by up to n_pub published frames (fewer when its images run out), all sequences
 * concurrently, and returns when every queue has drained (device work may still be in flight on the handles' streams).
 * Returns the number of published frames consumed over all sequences, or < 0 (a vt_status / ve_status value). */
int vr_advance(vr_session* s, int n_pub);

/* Per sequence counters since vr_open: published frames consumed, kernels launched, host<->device bytes. */
int vr_stats(const vr_session* s, int seq, int* frames, long long* launches, double* h2d_bytes, double* d2h_bytes);
/* Position of the newest window frame after every processImage in the NON_LINEAR state: copies up to cap entries,
 * returns the number available. */
int vr_trajectory(const vr_session* s, int seq, int cap, double* stamps, double* positions3);

/* Test access to the IMU side of the estimator loop (needs no device): for each of n_stamps image stamps, in order, the
 * (dt, acc, gyr) samples that would be handed to ve_process_imu before that image — getMeasurements' selection, the
 * per-sample dt and the interpolated sample at the stamp (estimator_node.cpp:98-136, 225-265).  counts[k] samples for
 * stamp k, concatenated in dt / acc_out / gyr_out (capacity cap samples).  Returns the total or < 0. */
int vr_debug_imu_batches(int n_imu, const double* imu_t, const double* acc, const double* gyr, int n_stamps, const double* stamps,
                         int cap, int* counts, double* dt, double* acc_out, double* gyr_out);

/* ---- The rest of the node shells (SURVEY.md 8f next-3), host only -----------------------------------------------------
 * High-rate pose prediction between two optimisations: estimator_node.cpp:42-78 predict() and :80-96 update().
 *   vr_prop_predict   one IMU message: the first one only latches its stamp (init_imu), later ones propagate tmp_P / tmp_Q /
 *                     tmp_V with the mid-point rule; out10 (may be NULL) receives P 3 | Q wxyz | V 3 (what pubLatestOdometry sends)
 *   vr_prop_update    update(): restart from the estimator's newest window state at `current_time` and re-apply the n queued
 *                     IMU messages (the node's imu_buf)
 *   vr_prop_update_from_estimator   the same, reading Ps/Rs/Vs/Bas/Bgs[WINDOW_SIZE], acc_0, gyr_0 and g from a handle */
typedef struct vr_propagator vr_propagator;
vr_propagator* vr_prop_create(void);
void vr_prop_destroy(vr_propagator* p);
int vr_prop_predict(vr_propagator* p, double t, const double* acc, const double* gyr, double* out10);
int vr_prop_update(vr_propagator* p, double current_time, const double* P3, const double* Qwxyz, const double* V3, const double* Ba3,
                   const double* Bg3, const double* acc0, const double* gyr0, const double* g3, int n, const double* t, const double* acc,
                   const double* gyr);
int vr_prop_update_from_estimator(vr_propagator* p, const ve_estimator* e, double current_time, int n, const double* t, const double* acc,
                                  const double* gyr);

/* One row of vins_result_no_loop.csv exactly as pubOdometry writes it (utility/visualization.cpp:156-172): the stamp in ns with
 * precision 0, then P, Q (w x y z), V with precision 5, every field followed by a comma, then a newline.  Returns the length
 * written (excluding the terminator) or < 0 when cap is too small. */
int vr_format_result_row(double stamp, const double* P3, const double* Qwxyz, const double* V3, char* buf, int cap);

/* Decoding of the tracker node's sensor_msgs/PointCloud into processImage's map (estimator_node.cpp:275-302): per point
 * v = id_of_point + 0.5, feature_id = v / NUM_OF_CAM, camera_id = v % NUM_OF_CAM (NUM_OF_CAM = 1), observation =
 * (x, y, z, u, v, velocity_x, velocity_y) widened to double; z must be 1 (ROS_ASSERT).  xyz: n x 3 float32.  Returns n or -1. */
int vr_decode_pointcloud(int n, const float* xyz, const float* id_of_point, const float* u_of_point, const float* v_of_point,
                         const float* velocity_x, const float* velocity_y, int* feature_ids, int* camera_ids, double* obs7);

/* Relocalisation messages (the pose_graph coupling; estimator_node.cpp:200-206, 266-291).
 *   vr_decode_relo_message   a /pose_graph/match_points PointCloud -> the arguments of setReloFrame: points (x, y, z = feature id)
 *                            -> match_points (n x 3 doubles); channels[0].values[0..2] = relo_t, [3..6] = relo_q (w x y z, turned
 *                            into relo_r like Quaterniond::toRotationMatrix, i.e. without normalising), [7] = frame_index; the
 *                            message's header stamp is the frame_stamp.  Returns n or -1.
 *   vr_queue_relo            puts a message into sequence seq's relo_buf with an arrival time: before the first image whose stamp is
 *                            >= arrival_stamp is processed, every message that has arrived is popped and the LAST one goes to
 *                            ve_set_relo_frame, exactly as process() does.  Call between vr_advance calls (not concurrently). */
int vr_decode_relo_message(int n, const float* xyz, const float* channel0_values8, double* match_points, double* relo_t3, double* relo_r9,
                           int* frame_index);
int vr_queue_relo(vr_session* s, int seq, double arrival_stamp, double frame_stamp, int frame_index, int n, const double* match_points,
                  const double* relo_t3, const double* relo_r9);

#ifdef __cplusplus
}
#endif
#endif
