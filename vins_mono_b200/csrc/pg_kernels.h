// Launch interface of the 4-DoF pose-graph solver (pg_kernels.cu).  Every launch serves a whole batch: the member slot
// is a grid dimension, the slots of this launch are listed in the header of the device input arena (pg_layout.h).
#pragma once
#include <cuda_runtime.h>

namespace vb {

struct PgLaunch {
    const char* d_in;    // device copy of the input arena (header + member blocks)
    double* d_work;      // member m's workspace at d_work + m * work_stride
    size_t work_stride;  // doubles
    double* d_out;       // output arena (member blocks at the header's out offsets)
    int S;               // batch size (header layout)
    int cap_n;           // key-frame capacity per member (workspace layout)
    int cap_anchors;     // free-anchor capacity per member (workspace layout)
    int count;           // active slots of this launch
    int max_n, max_D;    // maxima over the active slots (grid sizing)
    int max_iterations;
};

// Whole LM solve of every active slot: setup, max_iterations x {linearise, chain, border system, solve, update}, finish.
// When max_D > PG_MAX_D the border system and solve add the multi-CTA path: 2 ceil((max_D + 1) / 64) + 1 more launches
// per iteration.  Returns the number of kernels launched, or -1 when the device could not be configured for them (the CUDA error is
// left for cudaGetLastError).
int launch_pg_optimize(const PgLaunch& L, cudaStream_t s);
// Test access (vp_debug_four_dof_error): params8 = yaw_i, t_i, yaw_j, t_j; meas6 = t_rel, yaw_rel, pitch_i, roll_i;
// out = r[4] | J[4][8] | cost (0.5 rho), evaluated by the device code of the solve.
void launch_pg_debug_edge(const double* d_params8, const double* d_meas6, int weighted, int robust, double* d_out, cudaStream_t s);

}  // namespace vb
