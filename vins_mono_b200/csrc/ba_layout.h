// Layouts of the packed buffers of the batch BA path (ve_batch in estimator.cu): the per-frame input block, the output
// block, the states vector and the per-member device workspaces.  Each layout is defined here once, as offsets computed
// from the sizes it depends on; whatever sizes, carves, writes or reads one of these buffers goes through it.  Plain data
// and functions, usable from host code and from the kernels; tests/hostlib/ba_layout_host.cpp checks them with g++.
#pragma once
#include <cstddef>

#include "ba_types.h"

#ifdef __CUDACC__
#define BA_LAYOUT_FN __host__ __device__ constexpr inline
#else
#define BA_LAYOUT_FN constexpr inline
#endif

namespace vb {

BA_LAYOUT_FN size_t ba_align16(size_t bytes) { return (bytes + 15) & ~(size_t)15; }

// ---- states vector: one point x (BaStates), in doubles.  pose 7F | sb 9F | ex 7 | td 1 | lam L | relo_Pose 7 (+1)
struct BaStatesLayout {
    int pose, sb, ex, td, lam, relo, total;
};
BA_LAYOUT_FN BaStatesLayout ba_states_layout(int F, int L) {
    return BaStatesLayout{0, 7 * F, 16 * F, 16 * F + 7, 16 * F + 8, 16 * F + 8 + L, 16 * F + 8 + L + 8};
}
BA_LAYOUT_FN BaStates states_view(double* p, int F, int L) {
    const BaStatesLayout s = ba_states_layout(F, L);
    return BaStates{p + s.pose, p + s.sb, p + s.ex, p + s.td, p + s.lam, p + s.relo};
}

// ---- a member's output block, in doubles (written by ba_finish_kernel, read by the host after the frame):
//      SolverState | (W+1) x BA_OUT_FRAME (P, R row-major, V, Ba, Bg) | tic 3, ric 9 (row-major), td | L depths |
//      with a relocalisation block: relo_r 9 (row-major), relo_t 3
constexpr int BA_OUT_FRAME = 21, BA_OUT_EX = 13, BA_OUT_RELO = 12;
struct BaOutLayout {
    int frames, ex, depths, relo, total;
};
BA_LAYOUT_FN BaOutLayout ba_out_layout(int F, int L, bool relo) {
    return BaOutLayout{BA_OUT_ST_DOUBLES, BA_OUT_ST_DOUBLES + BA_OUT_FRAME * F, BA_OUT_ST_DOUBLES + BA_OUT_FRAME * F + BA_OUT_EX,
                       BA_OUT_ST_DOUBLES + BA_OUT_FRAME * F + BA_OUT_EX + L,
                       BA_OUT_ST_DOUBLES + BA_OUT_FRAME * F + BA_OUT_EX + L + (relo ? BA_OUT_RELO : 0)};
}
// doubles a block takes in the output arena: an even count, so the next block starts 16-byte aligned
BA_LAYOUT_FN size_t ba_out_reserve(int F, int L, bool relo) { return ((size_t)ba_out_layout(F, L, relo).total + 1) & ~(size_t)1; }

// ---- a member's input block of one frame, in bytes, every array 16-byte aligned:
//      pre-integration jobs | samples (7 doubles each) | int table | double table | states | marginalised landmark lists.
//      Without a solve the block holds the jobs and samples only.
struct BaInLayout {
    int W, L, M;
    size_t n_lm;
    size_t jobs, samples, ints, dbls, states, marg, total;
};
BA_LAYOUT_FN BaInLayout ba_in_layout(int W, size_t n_jobs, size_t n_rec, int L, int M, size_t n_lm, bool solve) {
    BaInLayout o{W, L, M, n_lm, 0, 0, 0, 0, 0, 0, 0};
    o.samples = ba_align16(n_jobs * sizeof(PreintJob));
    o.total = o.samples + ba_align16(n_rec * 7 * sizeof(double));
    if (solve) {
        o.ints = o.total;                                                                  // lm_anchor L | lm_start L+1 | ob_frame M | imu_slot W | lm_relo L
        o.dbls = o.ints + ba_align16(sizeof(int) * ((size_t)3 * L + 1 + M + W));        // lm_pts 2L | lm_vel 2L | lm_td L | lm_row L | ob_pts 2M | ob_vel 2M | ob_td M | ob_row M
        o.states = o.dbls + ba_align16(sizeof(double) * (6 * (size_t)L + 6 * (size_t)M));
        o.marg = o.states + ba_align16(sizeof(double) * ba_states_layout(W + 1, L).total);  // lms n_lm | col_lm n_lm
        o.total = o.marg + ba_align16(sizeof(int) * 2 * n_lm);
    }
    return o;
}
// At capacity (what the batch reserves for a member that may need it): 4 jobs per window frame, 4096 samples.
inline BaInLayout ba_in_layout_max(int W, int Lmax, int Mmax) {
    return ba_in_layout(W, (size_t)4 * (W + 1), 4096, Lmax, Mmax, (size_t)Lmax, true);
}

struct BaInPtrs {  // the input block's arrays at one base address (the pinned host block or its device copy)
    PreintJob* jobs;
    double* samples;
    int *lm_anchor, *lm_start, *ob_frame, *imu_slot, *lm_relo;
    double *lm_pts, *lm_vel, *lm_td, *lm_row, *ob_pts, *ob_vel, *ob_td, *ob_row;
    double* states;
    int *marg_lms, *marg_col_lm;
};
inline BaInPtrs ba_in_bind(unsigned char* base, const BaInLayout& o) {
    BaInPtrs p{};
    p.jobs = reinterpret_cast<PreintJob*>(base + o.jobs);
    p.samples = reinterpret_cast<double*>(base + o.samples);
    p.lm_anchor = reinterpret_cast<int*>(base + o.ints);
    p.lm_start = p.lm_anchor + o.L;
    p.ob_frame = p.lm_start + o.L + 1;
    p.imu_slot = p.ob_frame + o.M;
    p.lm_relo = p.imu_slot + o.W;
    p.lm_pts = reinterpret_cast<double*>(base + o.dbls);
    p.lm_vel = p.lm_pts + 2 * o.L;
    p.lm_td = p.lm_vel + 2 * o.L;
    p.lm_row = p.lm_td + o.L;
    p.ob_pts = p.lm_row + o.L;
    p.ob_vel = p.ob_pts + 2 * o.M;
    p.ob_td = p.ob_vel + 2 * o.M;
    p.ob_row = p.ob_td + o.M;
    p.states = reinterpret_cast<double*>(base + o.states);
    p.marg_lms = reinterpret_cast<int*>(base + o.marg);
    p.marg_col_lm = p.marg_lms + o.n_lm;
    return p;
}

// ---- per-member device workspaces, in doubles, sized once for the member's capacity (Lmax landmarks, Mmax
//      observation rows, D columns, priors of up to nmax parameters)

// linearisation records of one point (BaAccum), at the widest strides: obsJ | lmW | imuJ | gpr | gp | cost
struct BaAccLayout {
    size_t obsJ, lmW, imuJ, gpr, gp, cost, total;
};
BA_LAYOUT_FN BaAccLayout ba_acc_layout(int W, int Lmax, int Mmax, int D) {
    const size_t lmW = (size_t)Mmax * OJ_FULL, imuJ = lmW + (size_t)Lmax * LW_FULL, gpr = imuJ + (size_t)W * IMUJ_STRIDE,
                 gp = gpr + BA_PRIOR_COST + 8, cost = gp + D;
    return BaAccLayout{0, lmW, imuJ, gpr, gp, cost, cost + 8};
}

// a prior in information form (BaPrior): A nmax x nmax (used with leading dimension n) | g0 nmax | c0 | x0 9 per block
struct BaPriorLayout {
    size_t A, g0, c0, x0, total;
};
BA_LAYOUT_FN BaPriorLayout ba_prior_layout(int nmax) {
    const size_t g0 = (size_t)nmax * nmax;
    return BaPriorLayout{0, g0, g0 + nmax, g0 + nmax + 1, g0 + nmax + 1 + 9 * BA_MAX_PRIOR_BLOCKS};
}

// the marginalisation's dense system (MargPlan): Am P x P | bm P | Araw nmax x nmax | graw nmax + BA_MARG_DIAG (+1) |
// Wglobal (nmax + BA_MARG_MAX_DENSE)^2, with P = nmax + BA_MARG_MAX_DENSE + Lmax
struct BaMargLayout {
    size_t P, Am, bm, Araw, graw, Wglobal, total;
};
BA_LAYOUT_FN BaMargLayout ba_marg_layout(int nmax, int Lmax) {
    const size_t P = (size_t)nmax + BA_MARG_MAX_DENSE + Lmax, q = (size_t)nmax + BA_MARG_MAX_DENSE;
    const size_t bm = P * P, Araw = bm + P, graw = Araw + (size_t)nmax * nmax, Wglobal = graw + nmax + BA_MARG_DIAG + 1;
    return BaMargLayout{P, 0, bm, Araw, graw, Wglobal, Wglobal + q * q};
}

// the trust-region vectors of N = D + Lmax entries each: scale | diag | grad | gn
struct BaVecLayout {
    size_t scale, diag, grad, gn, total;
};
BA_LAYOUT_FN BaVecLayout ba_vec_layout(int D, int Lmax) {
    const size_t N = (size_t)D + Lmax;
    return BaVecLayout{0, N, 2 * N, 3 * N, 4 * N};
}

// ba_step_kernel's scratch for N = D + L: u | y | delta | (N unused) | the packed Cholesky factor of D + 1 rows (the last
// row carries the right-hand side).  The kernel evaluates it at the frame's D and L, the allocation at the capacity.
struct BaWorkLayout {
    size_t u, y, delta, Lp, total;
};
BA_LAYOUT_FN BaWorkLayout ba_work_layout(int D, int L) {
    const int N = D + L;
    return BaWorkLayout{0, (size_t)N, 2 * (size_t)N, 4 * (size_t)N, 4 * (size_t)N + (size_t)(D + 1) * (D + 2) / 2};
}

// The packed Schur complement (BaProblem::Spk): D (D + 1) / 2 doubles plus BA_SPK_SLACK, because ba_step_kernel's bulk
// copy moves whole 16-byte units and so rounds an odd count up by one double.
constexpr int BA_SPK_SLACK = 2;
BA_LAYOUT_FN size_t ba_spk_doubles(int D) { return (size_t)D * (D + 1) / 2 + BA_SPK_SLACK; }

}  // namespace vb
