// Launchers of the loop-verification kernels (lv_kernels.cu): key-frame attach (blur, FAST, BRIEF) and the verification
// of candidate pairs (BRIEF matching, PnP-RANSAC, relative pose).  Buffer layouts: lv_layout.h.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace vb {

// n_jobs key frames, job j: staging block j (lv_stage_layout) -> scratch j (lv_attach_layout) -> the arena slot at byte
// offset slots[j] (lv_slot_layout).  Blocks and scratches lie at their layout's total stride.  A slot is written only
// when its corner count fits max_corners; scratch status = {corner count, overflow}.
struct LvAttachLaunch {
    const char* stage;
    char* scratch;
    char* arena;
    const long long* slots;  // device, n_jobs slot byte offsets into the arena
    int n_jobs;
    const int* pattern;      // device, 256 x (x1, y1, x2, y2)
    int rows, cols, max_window, max_corners;
    double intrinsics[8];  // in the order of camera_model (camera_lift.h)
    int camera_model;      // CAM_PINHOLE, CAM_MEI or CAM_KANNALA_BRANDT
    double xi;             // MEI only
};
// ev (may be NULL): 4 events recorded before the blur, the FAST stage (FAST, compaction and the corner lift), BRIEF and
// after BRIEF.  Returns launches.
int launch_lv_attach(const LvAttachLaunch& L, cudaStream_t s, cudaEvent_t* ev);
// The corner lift alone: the status and the corners kp already in scratch and slots.
void launch_lv_lift(const LvAttachLaunch& L, cudaStream_t s);

// Loaded key frames into their slots (vp_load): staged (device) holds n_kf jobs and blocks as lv_load_layout defines them;
// each block's header, corners, normalised corners and descriptors go to its slot.  One launch.
void launch_lv_scatter(char* arena, const char* staged, int n_kf, int max_window, int max_corners, cudaStream_t s);

// n_jobs verifications.  jobs (device): per job the slot byte offsets of cur and old in the arena (2 x long long).
// Scratch (lv_conn_layout) and result (lv_result_doubles) per job at the given strides.
struct LvConnLaunch {
    const char* arena;
    const long long* jobs;
    char* scratch;
    size_t scratch_stride;
    double* result;
    size_t result_stride;
    int n_jobs, max_window, max_corners;
    double ric[9], tic[3];
};
// ev (may be NULL): 4 events before matching, the hypotheses, the refit and after it.  match = 0 skips the matching
// stage (scratch already holds the match list).  Returns launches.
int launch_lv_connect(const LvConnLaunch& L, cudaStream_t s, cudaEvent_t* ev, int match = 1);

}  // namespace vb
