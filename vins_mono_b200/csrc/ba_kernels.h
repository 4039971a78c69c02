// Launch interface of the BA kernels (ba_kernels.cu).  Every launch serves a whole batch: `seqs` is a device array of
// S per-member descriptors (ba_types.h), the member index is a grid dimension.
#pragma once
#include <cuda_runtime.h>

#include "ba_types.h"
#include "kprof.h"

namespace vb {

struct BatchShape {  // host-side maxima over the members of this frame: grid and shared-memory sizing
    int S;               // members
    int W;               // window size (uniform over the batch)
    int D;               // reduced dimension (uniform)
    int max_L;           // landmarks
    int max_n_lm;        // marginalised landmarks
    int max_md, max_n;   // marginalisation: dense marginalised columns, kept columns
    int max_P;           // marginalisation system size
    int any_jobs, any_active, any_marg;
    int any_relo;        // some member carries a relocalisation pose block this frame (its block pairs get CTAs)
    int est_ex, est_td;  // which optional parameter blocks are live (uniform over the batch: selects the kernel variants)
    int max_iterations;
    int w_in_global;     // marginalisation reduced system in global memory (decided once per batch: marg_w_in_global)
};

// profile slots: 0 eval (linearise), 1 reduce (Schur gather), 2 step, 3 unused, 4 marg zero + eval + gather, 5 marg_solve, 6 preint, 7 finish
// Pre-integration jobs (new slots, pushed samples, refreshed sqrt_info) of all members.
void launch_preint_jobs(BaSeq* seqs, const BatchShape& sh, cudaStream_t s, int* launches, KernelProfile* prof = nullptr);
// Full trust-region solve of every active member: linearise x[st.cur], then max_iterations x {schur, step,
// linearise + decide}; then the device-side double2vector / vector2double (results into the members' output blocks).
void launch_ba_solve(BaSeq* seqs, const BatchShape& sh, cudaStream_t s, int* launches, KernelProfile* prof = nullptr);
void launch_marginalize(BaSeq* seqs, const BatchShape& sh, cudaStream_t s, int* launches, KernelProfile* prof = nullptr);
// Whether marg_solve_kernel keeps its reduced system in global memory for these sizes on the current device.
int marg_w_in_global(int m_dense, int n);

// Test access (ve_debug_*): residual / Jacobian of single factors evaluated by the same device code as the solve.
// visual: out = r[2] | J[2][20]; imu: out = r_whitened[15] | Jw[15][30]
void launch_debug_visual(const BaDims& d, const double* d_params23, const double* d_data16, int robust, double* d_out, cudaStream_t s);
void launch_debug_imu(const BaDims& d, const PreInt* d_pre, const double* d_params32, double* d_out, cudaStream_t s);

}  // namespace vb
