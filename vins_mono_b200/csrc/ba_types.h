// Device-side data layout of the sliding-window BA path (all float64, structure-of-arrays in HBM).
//
// One "BaSeq" = one sequence's window at one frame: the problem (states current + candidate, the observation table
// grouped by landmark, the pre-integration slots, the marginalisation prior in information form, the accumulation
// buffers of the normal equations, the trust-region state), the pre-integration jobs of the frame, the gauge
// re-anchoring inputs of double2vector and the marginalisation plan.  A batch of S sequences is an array of S of
// these in device memory; every kernel takes the array and picks its member with a grid dimension, so one launch
// per stage serves the whole batch (S = 1 is the single-sequence path, the same code).
#pragma once
#include <cstdint>

namespace vb {

constexpr int BA_MAX_OBS_PER_LM = 32;  // lanes of the landmark warp (window size + 1 <= 32)
constexpr int BA_MAX_FRAMES = 32;
constexpr int BA_MAX_PRIOR_BLOCKS = 64;
// Capacity of the single-CTA solvers' work arrays, which fixes WINDOW_SIZE <= 22 (the reference ships 10):
constexpr int BA_MAX_D = 352;        // reduced (camera-side) system columns: 15 (W + 1) + 6 + 1 at W = 22
constexpr int BA_MAX_PRIOR_N = 160;  // prior parameters: 6 W + 9 + 6 + 1
constexpr int BA_MARG_MAX_DENSE = 15;  // marginalised non-landmark columns: a pose and a speed-bias block
constexpr int BA_MARG_DIAG = 7;        // diagnostics marg_solve_kernel writes behind the n entries of MargPlan::graw

struct PreInt {  // IntegrationBase (integration_base.h:189-209) + cached sqrt_info (imu_factor.h:64)
    double sum_dt;
    double dp[3], dq[4] /* w x y z */, dv[3];
    double ba[3], bg[3];      // linearized_ba / linearized_bg
    double acc0[3], gyr0[3];  // last sample (acc_0 / gyr_0)
    double jac[225], cov[225], sqrt_info[225];
};

struct BaDims {
    int W;        // WINDOW_SIZE; frames 0..W
    int D;        // reduced (camera-side) dimension: 6(W+1) + 9(W+1) [+6 ex] [+1 td] [+6 relo]
    int L;        // landmarks in this problem
    int M;        // non-anchor observations (= visual residual blocks)
    int est_ex, est_td;
    int col_sb;   // first speed-bias column = 6(W+1)
    int col_ex;   // -1 when the extrinsic is constant
    int col_td;   // -1 when td is not estimated
    int col_relo; // first column of the relocalisation pose block (relo_Pose, estimator.cpp:769-801), -1 without one
    int oj, lw;   // strides (doubles) of the per-observation / per-landmark linearisation records (BaAccum)
    double sqrt_info_vis;  // FOCAL_LENGTH / 1.5
    double tr_over_row;    // TR / ROW
    double half_row;       // ROW / 2 (projection_td_factor.cpp:18-19)
    double G[3];
};

struct BaStates {  // one point x: Ceres parameter layouts
    double* pose;  // (W+1) x 7: p, qx qy qz qw
    double* sb;    // (W+1) x 9: v, ba, bg
    double* ex;    // 7
    double* td;    // 1
    double* lam;   // L inverse depths
    double* relo;  // 7: relo_Pose (estimator.h:131), behind the inverse depths; only touched when dims.col_relo >= 0
};

// One linearisation point, factor by factor (nothing is accumulated with atomics: the normal equations are gathered
// from these records in a fixed order by ba_reduce_kernel, so a solve is bit-reproducible).  Record layouts:
//   obsJ  per visual residual block o (stride dims.oj):  Ji 2x6 | Jj 2x6 | r 2 | Jl 2 | wj = Jj^T Jl 6 | [Jex 2x6] [Jtd 2]
//   lmW   per landmark l (stride dims.lw), sums over its observations:
//         Hii = sum Ji^T Ji (21, packed upper) | gi = sum Ji^T r 6 | wi = sum Ji^T Jl 6 | Hll | gl | cost |
//         [Hie 6x6 | Hee 21 | ge 6 | we 6] [Hit 6 | Het 6 | Htt | gt | wt]
//   imuJ  per IMU factor k (stride 480): whitened Jacobian 15x30 | whitened residual 15 | cost | valid
//   gpr   prior gradient g0 + A dx (n <= BA_MAX_PRIOR_N), cost of the prior at gpr[BA_PRIOR_COST]
enum : int {
    OJ_JI = 0, OJ_JJ = 12, OJ_R = 24, OJ_JL = 26, OJ_WJ = 28, OJ_BASE = 34, OJ_JEX = 34, OJ_JTD = 46, OJ_FULL = 48,
    LW_HII = 0, LW_GI = 21, LW_WI = 27, LW_HLL = 33, LW_GL = 34, LW_COST = 35, LW_BASE = 36,
    LW_HIE = 36, LW_HEE = 72, LW_GE = 93, LW_WE = 99, LW_HIT = 105, LW_HET = 111, LW_HTT = 117, LW_GT = 118, LW_WT = 119, LW_FULL = 120,
    IMUJ_JW = 0, IMUJ_RW = 450, IMUJ_COST = 465, IMUJ_VALID = 466, IMUJ_STRIDE = 480,
    BA_PRIOR_COST = BA_MAX_PRIOR_N
};
struct BaAccum {
    double* obsJ;  // M x oj
    double* lmW;   // L x lw
    double* imuJ;  // W x IMUJ_STRIDE
    double* gpr;   // BA_PRIOR_COST + 8: n gradient entries, the prior's cost at gpr[BA_PRIOR_COST], padding
    double* gp;    // D: gradient of the camera-side parameters (written by ba_reduce_kernel)
    double* cost;  // 1: total cost, summed in a fixed order by the last CTA of ba_eval_kernel
};

struct BaPrior {  // MarginalizationInfo in information form: A = J0^T J0, g0 = J0^T r0, c0 = |r0|^2
    int n;            // rows/cols
    int nblocks;
    const int* type;  // per kept block: 0 pose, 1 speed-bias, 2 ex pose, 3 td
    const int* index; // frame index for pose / speed-bias blocks
    const int* off;   // local offset in the prior vector
    const double* x0; // nblocks x 9 linearization point (global parameterisation)
    const double* A;  // n x n
    const double* g0; // n
    const double* c0; // 1
};

struct SolverState {  // trust-region / dogleg state, lives in device memory
    int iteration, max_iterations;
    int done;        // 0 running; 1 iteration cap; 2 parameter tol; 3 function tol; 4 failure
    int cur;         // which of the two state/accumulation buffers holds the current point
    int reuse, cand_valid, first, successful, retries, invalid_streak;
    int alpha_valid, pad2;
    unsigned lin_ticket;
    int pad;
    double radius, mu, x_cost, cand_cost, model_cost_change, dogleg_step_norm, alpha, x_norm, step_norm;
    double initial_cost;
    long long clk[10];  // per-phase cycle counters of the last ba_step_kernel (profiling aid)
};
constexpr int BA_OUT_ST_DOUBLES = 32;  // room reserved for a SolverState at the head of a member's output block
static_assert(sizeof(SolverState) <= BA_OUT_ST_DOUBLES * sizeof(double), "output block header too small");

struct BaProblem {
    BaDims dims;
    BaStates x[2];
    BaAccum acc[2];
    // observation table
    const int* lm_anchor;     // L: frame of the first observation
    const int* lm_start;      // L+1: offsets into the ob_* arrays
    const double* lm_pts;     // L x 2: normalised point in the anchor frame (z = 1)
    const double* lm_vel;     // L x 2
    const double* lm_td;      // L
    const double* lm_row;     // L: raw v pixel coordinate
    const int* ob_frame;      // M (-1 for a relocalisation match: its "frame j" is relo_Pose)
    const int* lm_relo;       // L: 1 when the landmark's LAST observation row is its relocalisation match (read when col_relo >= 0)
    const double* ob_pts;     // M x 2
    const double* ob_vel;     // M x 2
    const double* ob_td;      // M
    const double* ob_row;     // M
    // IMU factors: factor k links frames k and k+1 through pre-integration slot imu_slot[k] (-1: skipped)
    PreInt* preint;           // slot array
    const int* imu_slot;      // W
    BaPrior prior;
    // solver workspace
    double* S;       // D x D Schur complement (full symmetric)
    double* Spk;     // the same, packed row-major lower triangle (what the Cholesky consumes)
    double* Hfull;   // D x D symmetrised Hpp
    double* gred;    // D
    double* scale;   // D + L Jacobi scaling
    double* diag;    // D + L trust-region diagonal
    double* grad;    // D + L
    double* gn;      // D + L
    double* work;    // step scratch and the packed Cholesky factor (ba_work_layout, ba_layout.h)
    SolverState* st; // points at BaSeq::st of the same member
};

struct MargPlan {  // dense marginalisation system layout: [m_dense | n_lm landmark columns | n kept]
    int P, m_dense, n_lm, n;
    const int* lms;     // device: indices (into the problem's landmark table) of the marginalised landmarks
    const int* col_lm;  // device: their columns
    int col_pose[BA_MAX_FRAMES], col_sb[BA_MAX_FRAMES];  // -1 when the block does not take part
    int col_ex, col_td;
    int use_imu;        // include IMU factor (frames 0,1)
    int w_in_global;    // the reduced system does not fit shared memory (set by the launcher, uniform per batch)
    double* Am;         // P x P (upper triangle accumulated)
    double* bm;         // P
    double* Aout;       // n x n   new prior A  (after the eps floor)
    double* gout;       // n       new prior g0
    double* cout;       // 1       new prior c0
    double* Araw;       // n x n   Schur complement before the eps floor (tests), may be null
    double* graw;       // n (+ BA_MARG_DIAG diagnostics)
    double* Wglobal;    // q x q scratch (q = m_dense + n) used when the reduced system does not fit shared memory
};

struct PreintJob {  // work of one frame on the pre-integration slots, executed in list order per slot
    int type;        // 0: new IntegrationBase{acc0, gyr0, ba, bg}; 1: push_back of n samples
    int slot, n, sample_off;  // sample_off in 7-double records (dt, acc[3], gyr[3]) from BaSeq::samples
    double acc0[3], gyr0[3], ba[3], bg[3];
};

// Inputs and outputs of the device-side double2vector + vector2double (estimator.cpp:530-619, :486-528) that runs
// between the solve and the marginalisation, so a frame needs no host round trip inside its kernel chain.
struct FinishPlan {
    double origin_ypr[3];  // R2ypr(Rs[0]) before the solve (degrees), or of last_R0 after a detected failure
    double origin_P0[3];
    double Rs0[9];         // Rs[0] before the solve (Euler-singularity fallback)
    double* out;           // member's output block (ba_out_layout, ba_layout.h); relo_r / relo_t: estimator.cpp:598-605
    int n_kept;            // kept blocks of the new prior (0: nothing is marginalised this frame)
    int kept_type[BA_MAX_PRIOR_BLOCKS], kept_index[BA_MAX_PRIOR_BLOCKS];  // pre-shift identities
    double* x0_out;        // new prior's linearisation point, 9 doubles per kept block
};

struct BaSeq {
    int active;            // this member runs a solve this frame
    int do_marg;           // ... and a marginalisation
    int n_jobs;
    unsigned sqrt_mask;    // slots whose sqrt_info is refreshed after the jobs
    const PreintJob* jobs;
    const double* samples;
    double noise[4];       // acc_n, gyr_n, acc_w, gyr_w
    int prior_type[BA_MAX_PRIOR_BLOCKS], prior_index[BA_MAX_PRIOR_BLOCKS], prior_off[BA_MAX_PRIOR_BLOCKS];
    SolverState st;
    BaProblem p;
    MargPlan mp;
    FinishPlan fin;
};

}  // namespace vb
