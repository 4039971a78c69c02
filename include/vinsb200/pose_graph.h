/* vinsb200 pose graph — C ABI of the 4-DoF pose-graph optimisation (pose_graph/src/pose_graph.h).
 *
 * Replaces, one entry point per reference interface:
 *   vp_create / vp_destroy     PoseGraph::PoseGraph (pose_graph.cpp:3-19) + the node's parameters
 *   vp_new_sequence            new_sequence() (pose_graph_node.cpp:69-72): the next key frame starts a new sequence
 *   vp_add_keyframe            PoseGraph::addKeyFrame (pose_graph.cpp:42-167) with findConnection's result passed in:
 *                              loop_index (-1: none) and loop_info8 = relative t (3), relative q (wxyz), relative yaw
 *                              (degrees); the loop is accepted through the gate |yaw| < 30 and |t| < 20
 *                              (keyframe.cpp:480).  Returns the stored (drift-corrected) pose.
 *   vp_update_loop             PoseGraph::updateKeyFrameLoop (pose_graph.cpp:889-923); loop_info8 laid out as
 *                              ve_get_relocalization returns it (relo_relative_t | relo_relative_q | relo_relative_yaw)
 *   vp_optimize                PoseGraph::optimize4DoF (pose_graph.cpp:403-579) for the newest key frame with an accepted
 *                              loop: enqueues the device solve and returns 1 (0 when nothing is pending)
 *   vp_correct_pose            the vio_callback transform (pose_graph_node.cpp:200-215): w_vio, then the drift
 *   vp_get_drift / vp_get_keyframe / vp_get_path   r_drift / t_drift / yaw_drift, one key frame, updatePath's list
 *
 * Asynchrony never changes results: vp_optimize enqueues and returns; the result is collected by the calls that read
 * poses or drift (vp_correct_pose, vp_get_*, vp_update_loop with fast relocalisation, vp_optimize itself) and by
 * vp_sync, which wait for it.  vp_add_keyframe never waits: it uses the drift of the last collected optimisation, as
 * addKeyFrame does while the reference's optimisation thread runs; key frames added after the optimised one are moved
 * by the new drift when the result is collected (pose_graph.cpp:562-571).
 *
 * Plain C, int status (0 ok, < 0 vp_status), no CPU fallback.  A handle is externally synchronised.  Capacity: at most
 * max_keyframes key frames, and at most max_anchors free loop anchors (distinct older key frames that loop edges land
 * on) in an optimised range; a call that would exceed either returns VP_ERR_CAPACITY and leaves the graph as it was.
 * Each anchor adds 4 columns to the dense border of the solve.  Borders up to 352 columns (88 anchors) are factored in
 * one CTA in shared memory; larger ones over many CTAs in global memory, on the FP64 tensor cores.  The device workspace
 * grows with max_anchors: per graph about 16 ceil(max_keyframes / 4) (4 max_anchors + 1) doubles for the chain's border
 * columns, plus (4 max_anchors + 1)^2 rounded up to 64 columns for the border system when max_anchors > 88; at 2048 key
 * frames and 1024 anchors that is about 268 MB + 138 MB.
 */
#ifndef VINSB200_POSE_GRAPH_H
#define VINSB200_POSE_GRAPH_H

#ifdef __cplusplus
extern "C" {
#endif

typedef enum vp_status { VP_OK = 0, VP_ERR_INVALID = -1, VP_ERR_NO_DEVICE = -2, VP_ERR_CUDA = -3, VP_ERR_CAPACITY = -4 } vp_status;

typedef struct vp_config {
    int max_keyframes;       /* key-frame capacity of the graph */
    int fast_relocalization; /* FAST_RELOCALIZATION (pose_graph_node.cpp, euroc_config.yaml:fast_relocalization) */
    int device;
    int max_anchors;         /* free-loop-anchor capacity of an optimised range: 0 = 88 (today's workspace), or 1 .. 1024;
                                anything else is VP_ERR_INVALID from vp_create / vp_batch_create */
} vp_config;

typedef struct vp_graph vp_graph;
typedef struct vp_batch vp_batch;

int vp_create(const vp_config* cfg, vp_graph** out);
void vp_destroy(vp_graph* g);
const char* vp_last_error(const vp_graph* g);

int vp_new_sequence(vp_graph* g);
/* index (may be NULL) = the key frame's global index; P3 / Qwxyz (may be NULL) = its stored pose */
int vp_add_keyframe(vp_graph* g, double stamp, const double* vio_P3, const double* vio_Qwxyz, int loop_index, const double* loop_info8,
                    int* index, double* P3, double* Qwxyz);
int vp_update_loop(vp_graph* g, int index, const double* loop_info8);

int vp_optimize(vp_graph* g);
int vp_sync(vp_graph* g);

/* P3 / Qwxyz in and out (in place allowed) */
int vp_correct_pose(vp_graph* g, const double* P3, const double* Qwxyz, double* P_out3, double* Q_out4);
/* r9 (row-major), t3, yaw (degrees); any pointer may be NULL */
int vp_get_drift(vp_graph* g, double* r9, double* t3, double* yaw);
/* vio14 = vio P (3) | vio Q wxyz (4) | P (3) | Q wxyz (4); loop_index (-1 none); loop_info8 */
int vp_get_keyframe(vp_graph* g, int index, double* vio14, int* loop_index, double* loop_info8);
/* every key frame: stamps, P (3), Q wxyz (4), sequence.  Returns the count; call with cap 0 for the count alone. */
int vp_get_path(vp_graph* g, int cap, double* stamps, double* P3, double* Qwxyz, int* sequence);
/* out8 = key frames, accepted loops, earliest_loop_index, optimisations run, and of the last optimisation: key frames,
 *        border columns, iterations, successful steps; costs2 = its initial and final cost */
int vp_info(vp_graph* g, int* out8, double* costs2);
/* device milliseconds (CUDA events) of the last collected optimisation; launches = kernels it launched */
int vp_last_timing(vp_graph* g, float* ms, int* launches);

/* ---- Batch: n independent graphs whose pending optimisations run in ONE launch chain (the member index is a grid
 * dimension), one host-to-device and one device-to-host copy for all of them.  A stand-alone handle from vp_create is a
 * batch of one running the same code.
 *   vp_batch_member      borrowed handle of member k for every per-graph call (not vp_destroy)
 *   vp_batch_optimize    vp_optimize for every member with active[k] != 0 (NULL = all); status[k] (may be NULL) = 1 when
 *                        member k was enqueued, 0 when it had nothing pending, < 0 on error; returns the first error or 0
 *   vp_batch_sync        collects every member's result
 *   vp_batch_last_timing device ms and launches of the last batch launch chain (wall ms includes the copies) */
int vp_batch_create(const vp_config* cfg, int n, vp_batch** out);
void vp_batch_destroy(vp_batch* b);
int vp_batch_size(const vp_batch* b);
vp_graph* vp_batch_member(vp_batch* b, int k);
const char* vp_batch_last_error(const vp_batch* b);
int vp_batch_optimize(vp_batch* b, const int* active, int* status);
int vp_batch_sync(vp_batch* b);
int vp_batch_last_timing(vp_batch* b, float* ms2, int* launches);

/* ---- Test entry: FourDOFError (weighted = 0) / FourDOFWeightError (weighted = 1, robust = 1 adds HuberLoss(0.1)) on the
 * device: params8 = yaw_i, t_i, yaw_j, t_j (degrees); meas6 = t_rel 3, yaw_rel, pitch_i, roll_i;
 * out37 = residual 4 | Jacobian 4 x 8 (yaw_i, t_i, yaw_j, t_j; row-major) | cost 0.5 rho. */
int vp_debug_four_dof_error(const double* params8, const double* meas6, int weighted, int robust, double* out37);

#ifdef __cplusplus
}
#endif
#endif
