// Linearisation and assembly of the sliding-window normal equations without atomics (included by ba_kernels.cu).
//
//   ba_eval_kernel     factor Evaluate() + Cauchy corrector (projection_factor.cpp:21-121, projection_td_factor.cpp:34-141,
//                      imu_factor.h:19-179, marginalization_factor.cpp:333-381), one warp per landmark (lanes = its
//                      observations), one CTA per IMU factor, one CTA for the prior.  Nothing is added into shared
//                      matrices: every factor leaves its Jacobian blocks in its own record (BaAccum), landmark sums are warp
//                      reductions.  The last CTA sums the cost in a fixed order and runs the trust-region accept/reject logic.
//   ba_reduce_kernel   Ceres' SchurEliminator restated as a gather: every 6x6 (pose, pose) block of
//                      S = Hpp - Hpl^T (Hll + mu E)^-1 Hpl is owned by one CTA that walks the landmarks seen from both frames
//                      IN ORDER (a feature track covers consecutive frames, so membership is two comparisons, no index lists);
//                      prior and IMU terms are added per entry in a fixed order.  Sparse (only co-visible landmarks are
//                      touched: ~6x fewer FLOPs than the dense L x D product) and bit-reproducible run to run.
#pragma once
#include "ba_device.cuh"

namespace vb {

constexpr int RED_THREADS = 256;

#define LIN_WARPS 4
__host__ __device__ inline int ba_eval_grid(const BaDims& d) { return (d.L + LIN_WARPS - 1) / LIN_WARPS + d.W + 1; }

// ---- trust-region bookkeeping after a point has been evaluated (Ceres TrustRegionMinimizer: iteration zero,
// ParameterToleranceReached, FunctionToleranceReached, IsStepSuccessful, Handle(Un)SuccessfulStep and
// DoglegStrategy::StepAccepted / StepRejected).
__device__ inline void decide(const BaProblem& p, int initial) {
    SolverState* st = p.st;
    if (initial) {
        const double c = *(volatile double*)p.acc[st->cur].cost;
        st->x_cost = c;
        st->initial_cost = c;
        return;
    }
    const double cand = *(volatile double*)p.acc[1 - st->cur].cost;
    st->cand_cost = cand;
    if (st->step_norm <= 1e-8 * (st->x_norm + 1e-8)) {
        st->done = 2;
        return;
    }
    const double cost_change = st->x_cost - cand;
    if (fabs(cost_change) <= 1e-6 * st->x_cost) {
        st->done = 3;
        return;
    }
    const double rho = cost_change / st->model_cost_change;
    if (rho > 1e-3) {
        st->cur = 1 - st->cur;
        st->x_cost = cand;
        st->successful++;
        if (rho < 0.25) st->radius *= 0.5;
        if (rho > 0.75) st->radius = fmax(st->radius, 3.0 * st->dogleg_step_norm);
        st->mu = fmax(1e-8, 2.0 * st->mu / 10.0);
        st->reuse = 0;
    } else {
        st->radius *= 0.5;
        st->reuse = 1;
    }
    if (st->iteration >= st->max_iterations) st->done = 1;
}

__device__ __forceinline__ int hii_index(int i, int j) { return i * 6 - i * (i - 1) / 2 + (j - i); }  // i <= j < 6, packed upper

// One landmark: lanes = its observations.  l_slot: record index of the landmark (== l for the solve; the marginalisation
// evaluates a subset and keeps the same indices).
// A relocalisation match (estimator.cpp:777-797) is the landmark's last observation row: a plain ProjectionFactor between the
// anchor pose and relo_Pose (no velocity / time-offset terms), evaluated by the last lane; the anchor-side sums below take it in
// like any other observation.  with_relo = false (the marginalisation, which never contains these factors) leaves the row out.
template <bool EX, bool TD>
__device__ __forceinline__ void lin_visual(const BaProblem& p, const BaStates& x, const BaAccum& a, int oj, int lw, int l, int lane,
                                           bool with_relo = true) {
    const BaDims& d = p.dims;
    const int s0 = p.lm_start[l], nrows = p.lm_start[l + 1] - s0;
    const int rl = d.col_relo >= 0 ? p.lm_relo[l] : 0;
    const int nobs = nrows - (with_relo ? 0 : rl);
    const int fi = p.lm_anchor[l];
    const bool has = lane < nobs;
    VisualEval e;
    if (has) {
        const int o = s0 + lane;
        const bool is_relo = rl != 0 && lane == nrows - 1;
        const double* pose_j = is_relo ? x.relo : x.pose + 7 * p.ob_frame[o];
        const double vs = is_relo ? 0.0 : 1.0;  // zero velocities: ProjectionTdFactor degenerates to ProjectionFactor
        eval_visual<EX, TD>(d, x.pose + 7 * fi, pose_j, x.ex, x.lam[l], d.est_td ? x.td[0] : 0.0, p.lm_pts[2 * l], p.lm_pts[2 * l + 1],
                            p.ob_pts[2 * o], p.ob_pts[2 * o + 1], vs * p.lm_vel[2 * l], vs * p.lm_vel[2 * l + 1], vs * p.ob_vel[2 * o],
                            vs * p.ob_vel[2 * o + 1], p.lm_td[l], p.ob_td[o], is_relo ? d.half_row : p.lm_row[l],
                            is_relo ? d.half_row : p.ob_row[o], true, true, e);
        double* rec = a.obsJ + (size_t)o * oj;
#pragma unroll
        for (int k = 0; k < 6; k++) {
            rec[OJ_JI + k] = e.J[0][k];
            rec[OJ_JI + 6 + k] = e.J[1][k];
            rec[OJ_JJ + k] = e.J[0][6 + k];
            rec[OJ_JJ + 6 + k] = e.J[1][6 + k];
            rec[OJ_WJ + k] = e.J[0][6 + k] * e.J[0][18] + e.J[1][6 + k] * e.J[1][18];
            if (EX) {
                rec[OJ_JEX + k] = e.J[0][12 + k];
                rec[OJ_JEX + 6 + k] = e.J[1][12 + k];
            }
        }
        rec[OJ_R] = e.r[0];
        rec[OJ_R + 1] = e.r[1];
        rec[OJ_JL] = e.J[0][18];
        rec[OJ_JL + 1] = e.J[1][18];
        if (TD) {
            rec[OJ_JTD] = e.J[0][19];
            rec[OJ_JTD + 1] = e.J[1][19];
        }
    } else {
        e.r[0] = e.r[1] = 0;
        e.half_rho = 0;
#pragma unroll
        for (int k = 0; k < 20; k++) e.J[0][k] = e.J[1][k] = 0;
    }
    double* out = a.lmW + (size_t)l * lw;
    auto dotJ = [&](int aa, int bb) { return e.J[0][aa] * e.J[0][bb] + e.J[1][aa] * e.J[1][bb]; };
    auto dotr = [&](int aa) { return e.J[0][aa] * e.r[0] + e.J[1][aa] * e.r[1]; };
    double v = warp_sum_d(e.half_rho);
    if (lane == 0) out[LW_COST] = v;
    v = warp_sum_d(dotJ(18, 18));
    if (lane == 0) out[LW_HLL] = v;
    v = warp_sum_d(dotr(18));
    if (lane == 0) out[LW_GL] = v;
    // blocks of the anchor pose (shared by all observations of the landmark): warp sums, lane 0 stores
#pragma unroll
    for (int aa = 0; aa < 6; aa++) {
#pragma unroll
        for (int bb = aa; bb < 6; bb++) {
            v = warp_sum_d(dotJ(aa, bb));
            if (lane == 0) out[LW_HII + hii_index(aa, bb)] = v;
        }
        v = warp_sum_d(dotr(aa));
        if (lane == 0) out[LW_GI + aa] = v;
        v = warp_sum_d(dotJ(aa, 18));
        if (lane == 0) out[LW_WI + aa] = v;
    }
    if (EX) {
#pragma unroll
        for (int aa = 0; aa < 6; aa++) {
#pragma unroll
            for (int bb = 0; bb < 6; bb++) {
                v = warp_sum_d(dotJ(aa, 12 + bb));
                if (lane == 0) out[LW_HIE + 6 * aa + bb] = v;
            }
#pragma unroll
            for (int bb = aa; bb < 6; bb++) {
                v = warp_sum_d(dotJ(12 + aa, 12 + bb));
                if (lane == 0) out[LW_HEE + hii_index(aa, bb)] = v;
            }
            v = warp_sum_d(dotr(12 + aa));
            if (lane == 0) out[LW_GE + aa] = v;
            v = warp_sum_d(dotJ(12 + aa, 18));
            if (lane == 0) out[LW_WE + aa] = v;
        }
    }
    if (TD) {
#pragma unroll
        for (int aa = 0; aa < 6; aa++) {
            v = warp_sum_d(dotJ(aa, 19));
            if (lane == 0) out[LW_HIT + aa] = v;
            v = warp_sum_d(EX ? dotJ(12 + aa, 19) : 0.0);
            if (lane == 0) out[LW_HET + aa] = v;
        }
        v = warp_sum_d(dotJ(19, 19));
        if (lane == 0) out[LW_HTT] = v;
        v = warp_sum_d(dotr(19));
        if (lane == 0) out[LW_GT] = v;
        v = warp_sum_d(dotJ(19, 18));
        if (lane == 0) out[LW_WT] = v;
    }
}

// One CTA per IMU factor: thread 0 evaluates the un-whitened residual and Jacobian blocks, then the CTA whitens them
// into the factor's record.
__device__ inline void lin_imu(const BaProblem& p, const BaStates& x, const BaAccum& a, int k, double* Jraw, double* rr) {
    const int tid = threadIdx.x, nt = blockDim.x;
    double* rec = a.imuJ + (size_t)k * IMUJ_STRIDE;
    const int slot = p.imu_slot[k];
    if (slot < 0) {
        if (tid == 0) {
            rec[IMUJ_VALID] = 0.0;
            rec[IMUJ_COST] = 0.0;
        }
        return;
    }
    const PreInt& pre = p.preint[slot];
    for (int i = tid; i < 450; i += nt) Jraw[i] = 0.0;
    __syncthreads();
    if (tid == 0) eval_imu_raw(p.dims, pre, x.pose + 7 * k, x.sb + 9 * k, x.pose + 7 * (k + 1), x.sb + 9 * (k + 1), rr, Jraw);
    __syncthreads();
    for (int idx = tid; idx < 450; idx += nt) {
        const int i = idx / 30, c = idx % 30;
        double s = 0;
        for (int q = 0; q < 15; q++) s += pre.sqrt_info[i * 15 + q] * Jraw[q * 30 + c];
        rec[IMUJ_JW + idx] = s;
    }
    if (tid < 15) {
        double s = 0;
        for (int q = 0; q < 15; q++) s += pre.sqrt_info[tid * 15 + q] * rr[q];
        rec[IMUJ_RW + tid] = s;
        Jraw[tid] = s;  // staged for the cost (Jraw is free again)
    }
    __syncthreads();
    if (tid == 0) {
        double c = 0;
        for (int q = 0; q < 15; q++) c += Jraw[q] * Jraw[q];
        rec[IMUJ_COST] = 0.5 * c;
        rec[IMUJ_VALID] = 1.0;
    }
}


// dx of the prior's kept blocks (MarginalizationFactor::Evaluate, marginalization_factor.cpp:343-364)
__device__ __forceinline__ void prior_dx(const BaProblem& p, const BaStates& x, double* dx, int tid, int nthreads) {
    const BaPrior& pr = p.prior;
    for (int b = tid; b < pr.nblocks; b += nthreads) {
        const int type = pr.type[b], idx = pr.index[b], off = pr.off[b];
        const double* x0 = pr.x0 + 9 * b;
        if (type == 0 || type == 2) {
            const double* xv = type == 0 ? x.pose + 7 * idx : x.ex;
            for (int q = 0; q < 3; q++) dx[off + q] = xv[q] - x0[q];
            const Quat dq = qmul(qinv(q_from_param(x0)), q_from_param(xv));
            const double sg = (dq.w >= 0) ? 2.0 : -2.0;
            dx[off + 3] = sg * dq.x;
            dx[off + 4] = sg * dq.y;
            dx[off + 5] = sg * dq.z;
        } else if (type == 1) {
            for (int q = 0; q < 9; q++) dx[off + q] = x.sb[9 * idx + q] - x0[q];
        } else {
            dx[off] = x.td[0] - x0[0];
        }
    }
}

// Prior: gradient g0 + A dx and cost 0.5 (c0 + dx^T (2 g0 + A dx)) into gpr (rows in a fixed order by one CTA).
__device__ inline void lin_prior(const BaProblem& p, const BaStates& x, const BaAccum& a, double* dx, double* red) {
    const BaPrior& pr = p.prior;
    const int n = pr.n, tid = threadIdx.x, nt = blockDim.x;
    if (n <= 0) {
        if (tid == 0) a.gpr[BA_PRIOR_COST] = 0.0;
        return;
    }
    prior_dx(p, x, dx, tid, nt);
    __syncthreads();
    const int lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    for (int aa = wid; aa < n; aa += nw) {  // a warp per row of A: coalesced reads, shuffle reduction
        double s = 0;
        for (int bb = lane; bb < n; bb += 32) s += pr.A[(size_t)aa * n + bb] * dx[bb];
        s = warp_sum_d(s);
        if (lane == 0) {
            s += pr.g0[aa];
            a.gpr[aa] = s;
            red[aa] = dx[aa] * (pr.g0[aa] + s);
        }
    }
    __syncthreads();
    if (tid < 32) {
        double c = 0;
        for (int i = lane; i < n; i += 32) c += red[i];
        c = warp_sum_d(c);
        if (lane == 0) a.gpr[BA_PRIOR_COST] = 0.5 * (pr.c0[0] + c);
    }
}

template <bool EX, bool TD>
__global__ void __launch_bounds__(32 * LIN_WARPS, 3) ba_eval_kernel(const BaSeq* __restrict__ seqs, int initial) {
    __shared__ double sJraw[450], srr[16];
    __shared__ double sdx[BA_MAX_PRIOR_N], sred[BA_MAX_PRIOR_N];
    __shared__ BaProblem sp;
    __shared__ int is_last;
    const BaSeq& q = seqs[blockIdx.y];
    if (!q.active) return;
    {
        const SolverState* st0 = &q.st;
        if (!initial && (st0->done || !st0->cand_valid)) return;
    }
    load_desc(&sp, &q.p);
    const BaProblem& p = sp;
    SolverState* st = p.st;
    const int grid = ba_eval_grid(p.dims);
    if ((int)blockIdx.x >= grid) return;  // the launch is sized for the largest member of the batch
    const int b = initial ? st->cur : 1 - st->cur;
    const BaStates x = p.x[b];
    const BaAccum a = p.acc[b];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int L = p.dims.L;
    const int nb_vis = (L + LIN_WARPS - 1) / LIN_WARPS, nb_imu = p.dims.W;
    const int blk = blockIdx.x;
    if (blk < nb_imu) {  // the long CTAs first
        lin_imu(p, x, a, blk, sJraw, srr);
    } else if (blk < nb_imu + nb_vis) {
        const int l = (blk - nb_imu) * LIN_WARPS + wid;
        if (l < L) lin_visual<EX, TD>(p, x, a, p.dims.oj, p.dims.lw, l, lane);
    } else {
        lin_prior(p, x, a, sdx, sred);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned t = atomicAdd(&st->lin_ticket, 1u);
        is_last = (t == (unsigned)grid - 1u);
    }
    __syncthreads();
    if (!is_last) return;
    // the last CTA to finish: total cost in a fixed order (prior, IMU factors, landmarks), then the step decision
    __threadfence();
    if (threadIdx.x < 32) {
        double c = 0;
        const volatile double* lmW = a.lmW;
        for (int l = lane; l < L; l += 32) c += lmW[(size_t)l * p.dims.lw + LW_COST];
        c = warp_sum_d(c);
        if (lane == 0) {
            double tot = ((const volatile double*)a.gpr)[BA_PRIOR_COST];
            for (int k = 0; k < nb_imu; k++) tot += ((const volatile double*)a.imuJ)[(size_t)k * IMUJ_STRIDE + IMUJ_COST];
            tot += c;
            *a.cost = tot;
            st->lin_ticket = 0;
            __threadfence();
            decide(p, initial);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Gather side.
// E_l = clamp(Hll_l s_l^2, 1e-6, 1e32) / s_l^2 is the dogleg/LM diagonal expressed in unscaled variables.
__device__ __forceinline__ double lm_inv_lambda(const BaProblem& p, const BaAccum& a, int l, double mu, int first) {
    const double h = a.lmW[(size_t)l * p.dims.lw + LW_HLL];
    const double s = first ? 1.0 / (1.0 + sqrt(h)) : p.scale[p.dims.D + l];
    const double d2 = fmin(fmax(h * s * s, 1e-6), 1e32);
    return 1.0 / (h + mu * d2 / (s * s));
}

struct ColInfo {  // a camera-side column: which parameter block it belongs to
    int type;     // 0 pose, 1 speed-bias, 2 ex, 3 td, 4 relocalisation pose
    int frame, i;
};
__device__ __forceinline__ ColInfo col_info(const BaDims& d, int c) {
    ColInfo ci;
    if (c < d.col_sb) {
        ci.type = 0;
        ci.frame = c / 6;
        ci.i = c - 6 * ci.frame;
    } else if (c < d.col_sb + 9 * (d.W + 1)) {
        ci.type = 1;
        ci.frame = (c - d.col_sb) / 9;
        ci.i = c - d.col_sb - 9 * ci.frame;
    } else if (d.col_relo >= 0 && c >= d.col_relo) {
        ci.type = 4;
        ci.frame = 0;
        ci.i = c - d.col_relo;
    } else if (d.col_ex >= 0 && c < d.col_ex + 6) {
        ci.type = 2;
        ci.frame = 0;
        ci.i = c - d.col_ex;
    } else {
        ci.type = 3;
        ci.frame = 0;
        ci.i = 0;
    }
    return ci;
}

// Local column (0..29) of a pose / speed-bias column inside IMU factor k, or -1.
__device__ __forceinline__ int imu_local(const ColInfo& c, int k) {
    if (c.type > 1) return -1;
    if (c.frame == k) return c.type == 0 ? c.i : 6 + c.i;
    if (c.frame == k + 1) return c.type == 0 ? 15 + c.i : 21 + c.i;
    return -1;
}

// J^T J entry (r, c) and gradient of the IMU factors, in factor order.
__device__ __forceinline__ double imu_entry(const BaDims& d, const BaAccum& a, const ColInfo& cr, const ColInfo& cc) {
    if (cr.type > 1 || cc.type > 1) return 0.0;
    const int k0 = min(cr.frame, cc.frame) - 1, k1 = min(cr.frame, cc.frame);
    double h = 0.0;
    for (int k = k0; k <= k1; k++) {
        if (k < 0 || k >= d.W) continue;
        const int la = imu_local(cr, k), lb = imu_local(cc, k);
        if (la < 0 || lb < 0) continue;
        const double* rec = a.imuJ + (size_t)k * IMUJ_STRIDE;
        if (rec[IMUJ_VALID] == 0.0) continue;
        double s = 0;
#pragma unroll
        for (int q = 0; q < 15; q++) s += rec[IMUJ_JW + q * 30 + la] * rec[IMUJ_JW + q * 30 + lb];
        h += s;
    }
    return h;
}
__device__ __forceinline__ double imu_grad(const BaDims& d, const BaAccum& a, const ColInfo& cr) {
    if (cr.type > 1) return 0.0;
    double g = 0.0;
    for (int k = cr.frame - 1; k <= cr.frame; k++) {
        if (k < 0 || k >= d.W) continue;
        const int la = imu_local(cr, k);
        const double* rec = a.imuJ + (size_t)k * IMUJ_STRIDE;
        if (la < 0 || rec[IMUJ_VALID] == 0.0) continue;
        double s = 0;
        for (int q = 0; q < 15; q++) s += rec[IMUJ_JW + q * 30 + la] * rec[IMUJ_RW + q];
        g += s;
    }
    return g;
}

// pinv[global column] = row of the prior, or -1
__device__ __forceinline__ void prior_inverse_map(const BaProblem& p, int* pinv, int tid, int nt) {
    const BaPrior& pr = p.prior;
    const BaDims& d = p.dims;
    for (int c = tid; c < d.D; c += nt) pinv[c] = -1;
    __syncthreads();
    for (int b = tid; b < pr.nblocks; b += nt) {
        const int type = pr.type[b], idx = pr.index[b], off = pr.off[b];
        if (type == 0) for (int q = 0; q < 6; q++) pinv[6 * idx + q] = off + q;
        else if (type == 1) for (int q = 0; q < 9; q++) pinv[d.col_sb + 9 * idx + q] = off + q;
        else if (type == 2) { if (d.col_ex >= 0) for (int q = 0; q < 6; q++) pinv[d.col_ex + q] = off + q; }
        else if (d.col_td >= 0) pinv[d.col_td] = off;
    }
    __syncthreads();
}
__device__ __forceinline__ double prior_entry(const BaPrior& pr, const int* pinv, int r, int c) {  // r <= c
    if (pr.n <= 0) return 0.0;
    const int aa = pinv[r], bb = pinv[c];
    return (aa >= 0 && bb >= 0) ? pr.A[(size_t)aa * pr.n + bb] : 0.0;
}

// "Pose-type" blocks: the parameter blocks visual factors touch.  T < F: pose of frame T; then [ex] [td] [relo], in this order.
struct VBlock {
    int type;  // 0 pose, 2 ex, 3 td, 4 relocalisation pose
    int frame, col, dim;
};
__device__ __forceinline__ int num_vblocks(const BaDims& d) {
    return d.W + 1 + (d.col_ex >= 0 ? 1 : 0) + (d.col_td >= 0 ? 1 : 0) + (d.col_relo >= 0 ? 1 : 0);
}
__device__ __forceinline__ VBlock vblock(const BaDims& d, int T) {
    const int F = d.W + 1;
    VBlock b;
    if (T < F) {
        b.type = 0; b.frame = T; b.col = 6 * T; b.dim = 6;
    } else if (d.col_relo >= 0 && T == num_vblocks(d) - 1) {
        b.type = 4; b.frame = 0; b.col = d.col_relo; b.dim = 6;
    } else if (d.col_ex >= 0 && T == F) {
        b.type = 2; b.frame = 0; b.col = d.col_ex; b.dim = 6;
    } else {
        b.type = 3; b.frame = 0; b.col = d.col_td; b.dim = 1;
    }
    return b;
}

// w_l restricted to block B, component i: J_B^T J_lambda summed over the landmark's observations.
// nobs = observations in window frames (the track); a relocalisation match, when the landmark has one, is row s0 + nobs.
__device__ __forceinline__ double lm_w(const BaAccum& a, int oj, const double* lw_rec, const VBlock& B, int i, int anchor, int s0, int nobs) {
    if (B.type == 0) return B.frame == anchor ? lw_rec[LW_WI + i] : a.obsJ[(size_t)(s0 + B.frame - anchor - 1) * oj + OJ_WJ + i];
    if (B.type == 2) return lw_rec[LW_WE + i];
    if (B.type == 4) return a.obsJ[(size_t)(s0 + nobs) * oj + OJ_WJ + i];
    return lw_rec[LW_WT];
}

// Visual J^T J entry (i, j) of block pair (A, B), A <= B in block order, contributed by landmark l (anchor, s0, nobs known to
// cover both blocks).
__device__ __forceinline__ double vis_entry(const BaAccum& a, int oj, const double* lw_rec, const VBlock& A, const VBlock& B, int i, int j,
                                            int anchor, int s0, int nobs) {
    if (B.type == 4) {  // relocalisation pose (always the last block): only the match's own factor links it to anything
        const double* o = a.obsJ + (size_t)(s0 + nobs) * oj;
        if (A.type == 0) return A.frame == anchor ? o[OJ_JI + i] * o[OJ_JJ + j] + o[OJ_JI + 6 + i] * o[OJ_JJ + 6 + j] : 0.0;
        if (A.type == 2) return o[OJ_JEX + i] * o[OJ_JJ + j] + o[OJ_JEX + 6 + i] * o[OJ_JJ + 6 + j];
        if (A.type == 3) return 0.0;  // a plain ProjectionFactor has no time-offset Jacobian
        return o[OJ_JJ + i] * o[OJ_JJ + j] + o[OJ_JJ + 6 + i] * o[OJ_JJ + 6 + j];
    }
    if (A.type == 0 && B.type == 0) {
        if (A.frame == B.frame) {
            if (A.frame == anchor) return lw_rec[LW_HII + (i <= j ? hii_index(i, j) : hii_index(j, i))];
            const double* o = a.obsJ + (size_t)(s0 + A.frame - anchor - 1) * oj;
            return o[OJ_JJ + i] * o[OJ_JJ + j] + o[OJ_JJ + 6 + i] * o[OJ_JJ + 6 + j];
        }
        if (A.frame != anchor) return 0.0;  // two non-anchor frames are not connected by a factor of this landmark
        const double* o = a.obsJ + (size_t)(s0 + B.frame - anchor - 1) * oj;
        return o[OJ_JI + i] * o[OJ_JJ + j] + o[OJ_JI + 6 + i] * o[OJ_JJ + 6 + j];
    }
    if (A.type == 0 && B.type == 2) {
        if (A.frame == anchor) return lw_rec[LW_HIE + 6 * i + j];
        const double* o = a.obsJ + (size_t)(s0 + A.frame - anchor - 1) * oj;
        return o[OJ_JJ + i] * o[OJ_JEX + j] + o[OJ_JJ + 6 + i] * o[OJ_JEX + 6 + j];
    }
    if (A.type == 0 && B.type == 3) {
        if (A.frame == anchor) return lw_rec[LW_HIT + i];
        const double* o = a.obsJ + (size_t)(s0 + A.frame - anchor - 1) * oj;
        return o[OJ_JJ + i] * o[OJ_JTD] + o[OJ_JJ + 6 + i] * o[OJ_JTD + 1];
    }
    if (A.type == 2 && B.type == 2) return lw_rec[LW_HEE + (i <= j ? hii_index(i, j) : hii_index(j, i))];
    if (A.type == 2 && B.type == 3) return lw_rec[LW_HET + i];
    return lw_rec[LW_HTT];
}
// Visual gradient component i of block A from landmark l.
__device__ __forceinline__ double vis_grad(const BaAccum& a, int oj, const double* lw_rec, const VBlock& A, int i, int anchor, int s0, int nobs) {
    if (A.type == 4) {
        const double* o = a.obsJ + (size_t)(s0 + nobs) * oj;
        return o[OJ_JJ + i] * o[OJ_R] + o[OJ_JJ + 6 + i] * o[OJ_R + 1];
    }
    if (A.type == 0) {
        if (A.frame == anchor) return lw_rec[LW_GI + i];
        const double* o = a.obsJ + (size_t)(s0 + A.frame - anchor - 1) * oj;
        return o[OJ_JJ + i] * o[OJ_R] + o[OJ_JJ + 6 + i] * o[OJ_R + 1];
    }
    if (A.type == 2) return lw_rec[LW_GE + i];
    return lw_rec[LW_GT];
}
__device__ __forceinline__ bool lm_covers(const VBlock& B, int anchor, int nobs, int rl) {
    if (B.type == 4) return rl != 0;
    return B.type != 0 || (anchor <= B.frame && B.frame <= anchor + nobs);
}

__device__ __forceinline__ void store_sym(const BaProblem& p, int r, int c, double h, double s) {  // r <= c
    const int D = p.dims.D;
    p.Hfull[(size_t)r * D + c] = h;
    p.S[(size_t)r * D + c] = s;
    p.Spk[(size_t)c * (c + 1) / 2 + r] = s;
    if (r != c) {
        p.Hfull[(size_t)c * D + r] = h;
        p.S[(size_t)c * D + r] = s;
    }
}

// grid.x: first the NV (NV + 1) / 2 pose-type block pairs (one CTA each), then CTAs of generic entries (4 per thread).
// A pair CTA first stages anchor / track length / record offset / 1/(Hll + mu E) of every landmark in shared memory (coalesced),
// so that the per-landmark terms need no dependent global loads: seven slices of 36 entry threads then walk the landmarks
// (slice s takes l = s, s + 7, ...) with predicated, unrolled loads from the factor records, and the slice sums are combined in a
// fixed order.
constexpr int RED_SLICES = 7;
constexpr int RED_SLAB = 1024;
// RELO = false is the kernel of frames without a relocalisation block (the usual case): no match-row bookkeeping at all.
template <bool RELO>
__global__ void __launch_bounds__(RED_THREADS, 3) ba_reduce_kernel(const BaSeq* __restrict__ seqs, int n_pairs_max) {
    __shared__ BaProblem sp;
    __shared__ int pinv[BA_MAX_D];
    __shared__ short s_an[RED_SLAB], s_nobs[RED_SLAB];
    __shared__ unsigned char s_rl[RED_SLAB];
    __shared__ int s_s0[RED_SLAB];
    __shared__ double s_inv[RED_SLAB];
    __shared__ double part[4][RED_SLICES][36];
    const BaSeq& q = seqs[blockIdx.y];
    if (!q.active || q.st.done || q.st.reuse) return;
    load_desc(&sp, &q.p);
    const BaProblem& p = sp;
    const BaDims& d = p.dims;
    const SolverState* st = p.st;
    const BaAccum a = p.acc[st->cur];
    const int tid = threadIdx.x, D = d.D, L = d.L, oj = d.oj, lw = d.lw;
    const int NV = num_vblocks(d), n_pairs = NV * (NV + 1) / 2;
    const double mu = st->mu;
    const int first = st->first;
    int blk = blockIdx.x;
    if (blk < n_pairs_max) {
        if (blk >= n_pairs) return;
        prior_inverse_map(p, pinv, tid, RED_THREADS);
        // pair index -> (TA <= TB): row TA holds pairs TB = TA .. NV-1
        int TA = 0, rem = blk;
        while (rem >= NV - TA) {
            rem -= NV - TA;
            TA++;
        }
        const int TB = TA + rem;
        const VBlock A = vblock(d, TA), B = vblock(d, TB);
        const int slice = tid / 36, e = tid - 36 * slice;  // threads 252..255 only help with the staging
        const int i = e / B.dim, j = e - i * B.dim;
        const bool worker = slice < RED_SLICES && e < A.dim * B.dim && !(TA == TB && i > j);
        const bool gworker = slice < RED_SLICES && TA == TB && e < A.dim;  // gradient component e of block A
        double h = 0.0, E = 0.0, gvis = 0.0, gE = 0.0;
        for (int l0 = 0; l0 < L; l0 += RED_SLAB) {
            const int nl = min(RED_SLAB, L - l0);
            __syncthreads();
            int unsorted = 0;
            for (int k = tid; k < nl; k += RED_THREADS) {
                const int l = l0 + k, s0 = p.lm_start[l];
                const int an = p.lm_anchor[l];
                const int rl = RELO && d.col_relo >= 0 ? p.lm_relo[l] : 0;
                s_an[k] = (short)an;
                s_nobs[k] = (short)(p.lm_start[l + 1] - s0 - rl);  // the track; a relocalisation match is the row behind it
                if (RELO) s_rl[k] = (unsigned char)rl;
                s_s0[k] = s0;
                s_inv[k] = lm_inv_lambda(p, a, l, mu, first);
                if (k > 0 && p.lm_anchor[l - 1] > an) unsorted = 1;
            }
            const int sorted_by_anchor = __syncthreads_or(unsorted) == 0;
            if ((worker || gworker) && A.type == 0 && B.type == 0) {
                // (pose a, pose b): the common case, written so that the loads of four landmarks are in flight together
                // (no early exits: uncovered landmarks contribute exact zeros through predicated loads)
                const int fa = A.frame, fb = B.frame;
                const bool diag = fa == fb;
                // The landmark table is ordered by anchor frame (FeatureManager appends new tracks at the end and the slides
                // keep the order), so the landmarks that can see frame a are a prefix [0, hi) of it.  hi is found from the
                // staged anchors; an unsorted table (never produced by the host) only costs the shortcut, not correctness.
                int hi = nl;
                if (sorted_by_anchor) {
                    int lo_ = 0, hi_ = nl;  // first k with anchor > fa
                    while (lo_ < hi_) {
                        const int mid = (lo_ + hi_) >> 1;
                        if (s_an[mid] <= fa) lo_ = mid + 1;
                        else hi_ = mid;
                    }
                    hi = lo_;
                }
                for (int k = slice; k < hi; k += 4 * RED_SLICES) {
                    double wa[4], wb[4], inv[4], x0[4], x1[4], y0[4], y1[4], gl[4], gv[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const int kk = k + u * RED_SLICES;
                        const bool in = kk < hi;
                        const int ks = in ? kk : 0;
                        const int an = s_an[ks], nobs = s_nobs[ks], s0 = s_s0[ks];
                        const bool cv = in && an <= fa && fb <= an + nobs;
                        const bool anchored = an == fa;
                        const double* rec = a.lmW + (size_t)(l0 + ks) * lw;
                        const double* oa = a.obsJ + (size_t)(s0 + max(fa - an - 1, 0)) * oj;  // observation in frame a (when not the anchor)
                        const double* ob = a.obsJ + (size_t)(s0 + max(fb - an - 1, 0)) * oj;  // observation in frame b
                        inv[u] = s_inv[ks];
                        wa[u] = cv ? (anchored ? rec[LW_WI + i] : oa[OJ_WJ + i]) : 0.0;
                        wb[u] = cv ? ((an == fb) ? rec[LW_WI + j] : ob[OJ_WJ + j]) : 0.0;
                        gl[u] = cv ? rec[LW_GL] : 0.0;
                        if (diag) {
                            // anchored: Hii(i, j); otherwise Jj^T Jj of the observation in this frame
                            const int hij = i <= j ? hii_index(i, j) : hii_index(j, i);
                            x0[u] = cv ? (anchored ? rec[LW_HII + hij] : oa[OJ_JJ + i]) : 0.0;
                            y0[u] = cv && !anchored ? oa[OJ_JJ + j] : (anchored ? 1.0 : 0.0);
                            x1[u] = cv && !anchored ? oa[OJ_JJ + 6 + i] : 0.0;
                            y1[u] = cv && !anchored ? oa[OJ_JJ + 6 + j] : 0.0;
                            // gradient threads are the entries (0, e): their component index is j
                            gv[u] = cv ? (anchored ? rec[LW_GI + j] : oa[OJ_JJ + j] * oa[OJ_R] + oa[OJ_JJ + 6 + j] * oa[OJ_R + 1]) : 0.0;
                        } else {
                            const bool on = cv && anchored;  // only the factor anchored in a links a and b
                            x0[u] = on ? ob[OJ_JI + i] : 0.0;
                            y0[u] = on ? ob[OJ_JJ + j] : 0.0;
                            x1[u] = on ? ob[OJ_JI + 6 + i] : 0.0;
                            y1[u] = on ? ob[OJ_JJ + 6 + j] : 0.0;
                            gv[u] = 0.0;
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        if (worker) {
                            h += x0[u] * y0[u] + x1[u] * y1[u];
                            E += wa[u] * inv[u] * wb[u];
                        }
                        if (gworker) {  // diagonal pair: block B is block A, so wb is component j = e of w_A
                            gvis += gv[u];
                            gE += wb[u] * inv[u] * gl[u];
                        }
                    }
                }
            } else if (worker || gworker) {
#pragma unroll 4
                for (int k = slice; k < nl; k += RED_SLICES) {
                    const int an = s_an[k], nobs = s_nobs[k], s0 = s_s0[k], rl = RELO ? s_rl[k] : 0;
                    if (!lm_covers(A, an, nobs, rl) || !lm_covers(B, an, nobs, rl)) continue;
                    const double* rec = a.lmW + (size_t)(l0 + k) * lw;
                    const double inv = s_inv[k];
                    if (worker) {
                        h += vis_entry(a, oj, rec, A, B, i, j, an, s0, nobs);
                        E += lm_w(a, oj, rec, A, i, an, s0, nobs) * inv * lm_w(a, oj, rec, B, j, an, s0, nobs);
                    }
                    if (gworker) {
                        gvis += vis_grad(a, oj, rec, A, e, an, s0, nobs);
                        gE += lm_w(a, oj, rec, A, e, an, s0, nobs) * inv * rec[LW_GL];
                    }
                }
            }
        }
        if (slice < RED_SLICES) {
            part[0][slice][e] = h;
            part[1][slice][e] = E;
            part[2][slice][e] = gvis;
            part[3][slice][e] = gE;
        }
        __syncthreads();
        if (slice == 0 && worker) {
            const int r = A.col + i, c = B.col + j;
            const double base = prior_entry(p.prior, pinv, r, c) + imu_entry(d, a, col_info(d, r), col_info(d, c));
            double hs = part[0][0][e], Ev = part[1][0][e];
#pragma unroll
            for (int sl = 1; sl < RED_SLICES; sl++) {  // slices in order
                hs += part[0][sl][e];
                Ev += part[1][sl][e];
            }
            const double hv = base + hs;
            store_sym(p, r, c, hv, hv - Ev);
        }
        if (slice == 0 && gworker) {
            const int rg = A.col + e;
            const double gbase = (p.prior.n > 0 && pinv[rg] >= 0 ? a.gpr[pinv[rg]] : 0.0) + imu_grad(d, a, col_info(d, rg));
            double gs = part[2][0][e], gEs = part[3][0][e];
#pragma unroll
            for (int sl = 1; sl < RED_SLICES; sl++) {
                gs += part[2][sl][e];
                gEs += part[3][sl][e];
            }
            const double g = gbase + gs;
            a.gp[rg] = g;
            p.gred[rg] = g - gEs;
        }
        return;
    }
    // generic entries: everything that involves a speed-bias column (prior + IMU terms only)
    blk -= n_pairs_max;
    prior_inverse_map(p, pinv, tid, RED_THREADS);
    const int total = D * (D + 1) / 2;
    for (int e = 0; e < 4; e++) {
        const int idx = (blk * 4 + e) * RED_THREADS + tid;
        if (idx >= total) break;
        int c = (int)((sqrtf(8.f * (float)idx + 1.f) - 1.f) * 0.5f);
        while (c * (c + 1) / 2 > idx) c--;
        while ((c + 1) * (c + 2) / 2 <= idx) c++;
        const int r = idx - c * (c + 1) / 2;  // r <= c
        const ColInfo cr = col_info(d, r), cc = col_info(d, c);
        if (cr.type != 1 && cc.type != 1) continue;  // owned by a block-pair CTA
        const double h = prior_entry(p.prior, pinv, r, c) + imu_entry(d, a, cr, cc);
        store_sym(p, r, c, h, h);
        if (r == c) {
            const double g = (p.prior.n > 0 && pinv[r] >= 0 ? a.gpr[pinv[r]] : 0.0) + imu_grad(d, a, cr);
            a.gp[r] = g;
            p.gred[r] = g;
        }
    }
}

// sum over the camera-side columns a landmark touches of w_l[c] v[c], by one warp (fixed lane assignment + shuffle tree)
__device__ __forceinline__ double lm_row_dot(const BaProblem& p, const BaAccum& a, int l, const double* v, int lane) {
    const BaDims& d = p.dims;
    const int rl = d.col_relo >= 0 ? p.lm_relo[l] : 0;
    const int an = p.lm_anchor[l], s0 = p.lm_start[l], nobs = p.lm_start[l + 1] - s0 - rl;
    const double* rec = a.lmW + (size_t)l * d.lw;
    double s = 0;
    for (int idx = lane; idx < 6 * (nobs + 1); idx += 32) {
        const int t = idx / 6, i = idx - 6 * t;
        const double w = t == 0 ? rec[LW_WI + i] : a.obsJ[(size_t)(s0 + t - 1) * d.oj + OJ_WJ + i];
        s += w * v[6 * (an + t) + i];
    }
    if (rl && lane >= 8 && lane < 14) s += a.obsJ[(size_t)(s0 + nobs) * d.oj + OJ_WJ + lane - 8] * v[d.col_relo + lane - 8];
    if (d.col_ex >= 0 && lane < 6) s += rec[LW_WE + lane] * v[d.col_ex + lane];
    if (d.col_td >= 0 && lane == 6) s += rec[LW_WT] * v[d.col_td];
    return warp_sum_d(s);
}

// The same sum by a group of 8 adjacent lanes (gl = lane within the group); every lane of the warp must call it (l >= L: 0).
__device__ __forceinline__ double lm_row_dot8(const BaProblem& p, const BaAccum& a, int l, int L, const double* v, int gl) {
    const BaDims& d = p.dims;
    double s = 0;
    if (l < L) {
        const int rl = d.col_relo >= 0 ? p.lm_relo[l] : 0;
        const int an = p.lm_anchor[l], s0 = p.lm_start[l], nobs = p.lm_start[l + 1] - s0 - rl;
        const double* rec = a.lmW + (size_t)l * d.lw;
        for (int idx = gl; idx < 6 * (nobs + 1); idx += 8) {
            const int t = idx / 6, i = idx - 6 * t;
            const double w = t == 0 ? rec[LW_WI + i] : a.obsJ[(size_t)(s0 + t - 1) * d.oj + OJ_WJ + i];
            s += w * v[6 * (an + t) + i];
        }
        if (rl && gl < 6) s += a.obsJ[(size_t)(s0 + nobs) * d.oj + OJ_WJ + gl] * v[d.col_relo + gl];
        if (d.col_ex >= 0 && gl < 6) s += rec[LW_WE + gl] * v[d.col_ex + gl];
        if (d.col_td >= 0 && gl == 6) s += rec[LW_WT] * v[d.col_td];
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    return s;
}

}  // namespace vb
