// Sliding-window BA kernels for sm_90a (SURVEY.md §8 rows b1, b5-b11, b13), float64.
//
//   preint_push_kernel    IntegrationBase::propagate / midPointIntegration     integration_base.h:54-158
//   sqrt_info_kernel      LLT(covariance^-1).matrixL().transpose()            imu_factor.h:64
//   ba_eval_kernel        factor Evaluate() + Cauchy corrector into per-factor records (ba_assemble.cuh); the last CTA to
//                         finish runs the trust-region accept/reject logic
//   ba_reduce_kernel      landmark elimination S = Hpp - Hpl^T (Hll + mu E)^-1 Hpl gathered block by block in a fixed
//                         order (no atomics, only co-visible landmarks), plus the reduced gradient
//   ba_step_kernel        Jacobi scaling, dogleg (Cauchy point, regularised Gauss-Newton via in-shared-memory
//                         Cholesky), model cost change, candidate point x (+) delta
//   marg_eval / marg_gather / marg_solve_kernel   MarginalizationInfo::preMarginalize + marginalize
//                         (marginalization_factor.cpp:110-297) producing the new prior in information form
// The solve replaces ceres::Solve(DENSE_SCHUR, DOGLEG) at estimator.cpp:803-818; no wall-clock cap.
// Everything here is small dense float64 algebra: latency bound for one sequence, HBM bound in batches;
// the FP64 pipe is far from saturated, so no tensor-core path is used (see DESIGN.md).
#include "ba_kernels.h"
#include "ba_layout.h"
#include "cuda_check.h"

#include <algorithm>
#include <map>
#include <mutex>
#include <cfloat>

#include "ba_device.cuh"
#include "prior_floor.h"

namespace vb {

// ------------------------------------------------------------------------------------------------
// IMU pre-integration: appends n samples (dt, acc[3], gyr[3]) to one slot.  Single CTA of 256 threads;
// the 15x15 products run in parallel, the 3x3 geometry of each step on thread 0.
struct PreintSmem {
    double F[225], V[270], J[225], P[225], T[225], nz[18];
    double st[20];  // dp dq dv acc0 gyr0
};
__device__ void preint_push_dev(PreInt* __restrict__ slot, int n, const double* __restrict__ samples, double acc_n, double gyr_n,
                                double acc_w, double gyr_w, PreintSmem& sm) {
    double *F = sm.F, *V = sm.V, *J = sm.J, *P = sm.P, *T = sm.T, *nz = sm.nz, *st = sm.st;
    const int tid = threadIdx.x;
    __syncthreads();  // the previous job of this CTA is done with the shared arrays
    for (int i = tid; i < 225; i += 256) {
        J[i] = slot->jac[i];
        P[i] = slot->cov[i];
    }
    if (tid < 18) nz[tid] = tid < 3 ? acc_n * acc_n : tid < 6 ? gyr_n * gyr_n : tid < 9 ? acc_n * acc_n : tid < 12 ? gyr_n * gyr_n : tid < 15 ? acc_w * acc_w : gyr_w * gyr_w;
    if (tid == 0) {
        for (int i = 0; i < 3; i++) { st[i] = slot->dp[i]; st[7 + i] = slot->dv[i]; st[10 + i] = slot->acc0[i]; st[13 + i] = slot->gyr0[i]; }
        for (int i = 0; i < 4; i++) st[3 + i] = slot->dq[i];
        st[16] = slot->sum_dt;
    }
    __syncthreads();
    const Vec3 ba = Vec3(slot->ba[0], slot->ba[1], slot->ba[2]), bg = Vec3(slot->bg[0], slot->bg[1], slot->bg[2]);
    for (int k = 0; k < n; k++) {
        for (int i = tid; i < 225; i += 256) F[i] = 0.0;
        for (int i = tid; i < 270; i += 256) V[i] = 0.0;
        __syncthreads();
        if (tid == 0) {
            const double dt = samples[7 * k];
            const Vec3 a1 = Vec3(samples[7 * k + 1], samples[7 * k + 2], samples[7 * k + 3]);
            const Vec3 g1 = Vec3(samples[7 * k + 4], samples[7 * k + 5], samples[7 * k + 6]);
            const Vec3 a0 = Vec3(st[10], st[11], st[12]), g0 = Vec3(st[13], st[14], st[15]);
            const Vec3 dp = Vec3(st[0], st[1], st[2]), dv = Vec3(st[7], st[8], st[9]);
            const Quat dq = Quat{st[3], st[4], st[5], st[6]};
            const Vec3 un_acc_0 = qrot(dq, a0 - ba);
            const Vec3 un_gyr = 0.5 * (g0 + g1) - bg;
            const Quat rq = qmul(dq, Quat{1, un_gyr.x * dt / 2, un_gyr.y * dt / 2, un_gyr.z * dt / 2});
            const Vec3 un_acc_1 = qrot(rq, a1 - ba);
            const Vec3 un_acc = 0.5 * (un_acc_0 + un_acc_1);
            const Vec3 rdp = dp + dv * dt + 0.5 * un_acc * dt * dt;
            const Vec3 rdv = dv + un_acc * dt;
            const Mat3 Rwx = skew(un_gyr), Ra0 = skew(a0 - ba), Ra1 = skew(a1 - ba);
            const Mat3 Rq = qR(dq), Rr = qR(rq), I = Mat3();
            const Mat3 ImW = msub(I, mscale(Rwx, dt));
            auto putF = [&](int r0, int c0, const Mat3& b) { for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) F[(r0 + i) * 15 + c0 + j] = b.m[3 * i + j]; };
            auto putV = [&](int r0, int c0, const Mat3& b) { for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) V[(r0 + i) * 18 + c0 + j] = b.m[3 * i + j]; };
            const Mat3 RqA0 = mmul(Rq, Ra0), RrA1 = mmul(Rr, Ra1), RrA1W = mmul(RrA1, ImW);
            putF(0, 0, I);
            putF(0, 3, madd(mscale(RqA0, -0.25 * dt * dt), mscale(RrA1W, -0.25 * dt * dt)));
            putF(0, 6, mscale(I, dt));
            putF(0, 9, mscale(madd(Rq, Rr), -0.25 * dt * dt));
            putF(0, 12, mscale(RrA1, -0.25 * dt * dt * -dt));
            putF(3, 3, ImW);
            putF(3, 12, mscale(I, -1.0 * dt));
            putF(6, 3, madd(mscale(RqA0, -0.5 * dt), mscale(RrA1W, -0.5 * dt)));
            putF(6, 6, I);
            putF(6, 9, mscale(madd(Rq, Rr), -0.5 * dt));
            putF(6, 12, mscale(RrA1, -0.5 * dt * -dt));
            putF(9, 9, I);
            putF(12, 12, I);
            const Mat3 v03 = mscale(RrA1, 0.25 * -1.0 * dt * dt * 0.5 * dt), v63 = mscale(RrA1, 0.5 * -1.0 * dt * 0.5 * dt);
            putV(0, 0, mscale(Rq, 0.25 * dt * dt));
            putV(0, 3, v03);
            putV(0, 6, mscale(Rr, 0.25 * dt * dt));
            putV(0, 9, v03);
            putV(3, 3, mscale(I, 0.5 * dt));
            putV(3, 9, mscale(I, 0.5 * dt));
            putV(6, 0, mscale(Rq, 0.5 * dt));
            putV(6, 3, v63);
            putV(6, 6, mscale(Rr, 0.5 * dt));
            putV(6, 9, v63);
            putV(9, 12, mscale(I, dt));
            putV(12, 15, mscale(I, dt));
            const Quat nq = qnormalized(rq);
            st[0] = rdp.x; st[1] = rdp.y; st[2] = rdp.z;
            st[3] = nq.w; st[4] = nq.x; st[5] = nq.y; st[6] = nq.z;
            st[7] = rdv.x; st[8] = rdv.y; st[9] = rdv.z;
            st[10] = a1.x; st[11] = a1.y; st[12] = a1.z;
            st[13] = g1.x; st[14] = g1.y; st[15] = g1.z;
            st[16] += dt;
        }
        __syncthreads();
        if (tid < 225) {  // T = F * J ; then J = T
            const int i = tid / 15, j = tid % 15;
            double s = 0;
            for (int q = 0; q < 15; q++) s += F[i * 15 + q] * J[q * 15 + j];
            T[tid] = s;
        }
        __syncthreads();
        if (tid < 225) J[tid] = T[tid];
        __syncthreads();
        if (tid < 225) {  // T = F * P
            const int i = tid / 15, j = tid % 15;
            double s = 0;
            for (int q = 0; q < 15; q++) s += F[i * 15 + q] * P[q * 15 + j];
            T[tid] = s;
        }
        __syncthreads();
        if (tid < 225) {  // P = T * F^T + V N V^T
            const int i = tid / 15, j = tid % 15;
            double s = 0;
            for (int q = 0; q < 15; q++) s += T[i * 15 + q] * F[j * 15 + q];
            double v = 0;
            for (int q = 0; q < 18; q++) v += V[i * 18 + q] * nz[q] * V[j * 18 + q];
            P[tid] = s + v;
        }
        __syncthreads();
    }
    for (int i = tid; i < 225; i += 256) {
        slot->jac[i] = J[i];
        slot->cov[i] = P[i];
    }
    if (tid == 0) {
        for (int i = 0; i < 3; i++) { slot->dp[i] = st[i]; slot->dv[i] = st[7 + i]; slot->acc0[i] = st[10 + i]; slot->gyr0[i] = st[13 + i]; }
        for (int i = 0; i < 4; i++) slot->dq[i] = st[3 + i];
        slot->sum_dt = st[16];
    }
    __threadfence_block();
    __syncthreads();  // the slot is complete in global memory before the next job (or the sqrt_info refresh) reads it
}

// new IntegrationBase{acc_0, gyr_0, ba, bg}: identity Jacobian, zero covariance (integration_base.h:13-28)
__device__ void preint_init_dev(PreInt* __restrict__ slot, const PreintJob& v) {
    const int tid = threadIdx.x;
    __syncthreads();
    for (int i = tid; i < 225; i += 256) {
        slot->jac[i] = (i / 15 == i % 15) ? 1.0 : 0.0;
        slot->cov[i] = 0.0;
        slot->sqrt_info[i] = 0.0;
    }
    if (tid == 0) {
        slot->sum_dt = 0.0;
        slot->dq[0] = 1.0;
        for (int i = 0; i < 3; i++) {
            slot->dp[i] = 0.0;
            slot->dv[i] = 0.0;
            slot->dq[1 + i] = 0.0;
            slot->ba[i] = v.ba[i];
            slot->bg[i] = v.bg[i];
            slot->acc0[i] = v.acc0[i];
            slot->gyr0[i] = v.gyr0[i];
        }
    }
    __threadfence_block();
    __syncthreads();
}

// sqrt_info = chol_lower(cov^-1)^T for each listed slot (one warp each; Gauss-Jordan with partial pivoting).
// Runs on the first warp of the CTA.
__device__ void sqrt_info_dev(PreInt* __restrict__ s, double (*A)[31], double (*Lm)[15]) {
    const int lane = threadIdx.x;
    for (int i = lane; i < 225; i += 32) {
        A[i / 15][i % 15] = s->cov[i];
        A[i / 15][15 + i % 15] = (i / 15 == i % 15) ? 1.0 : 0.0;
    }
    __syncwarp();
    for (int k = 0; k < 15; k++) {
        int piv = k;
        double best = fabs(A[k][k]);
        for (int i = k + 1; i < 15; i++)
            if (fabs(A[i][k]) > best) best = fabs(A[i][k]), piv = i;
        if (piv != k && lane < 30) {
            const double t = A[k][lane];
            A[k][lane] = A[piv][lane];
            A[piv][lane] = t;
        }
        __syncwarp();
        const double pv = A[k][k];
        __syncwarp();
        if (lane < 30) A[k][lane] /= pv;
        __syncwarp();
        for (int i = 0; i < 15; i++) {
            if (i == k) continue;
            const double f = A[i][k];
            __syncwarp();
            if (lane < 30) A[i][lane] -= f * A[k][lane];
            __syncwarp();
        }
    }
    // A[:,15:30] = cov^-1 ; lower Cholesky
    for (int j = 0; j < 15; j++) {
        double sdiag = A[j][15 + j];
        for (int k = 0; k < j; k++) sdiag -= Lm[j][k] * Lm[j][k];
        const double ljj = sqrt(sdiag);
        __syncwarp();
        if (lane == 0) Lm[j][j] = ljj;
        if (lane > j && lane < 15) {
            double t = 0.5 * (A[lane][15 + j] + A[j][15 + lane]);
            for (int k = 0; k < j; k++) t -= Lm[lane][k] * Lm[j][k];
            Lm[lane][j] = t / ljj;
        }
        if (lane < j) Lm[lane][j] = 0.0;
        __syncwarp();
    }
    for (int i = lane; i < 225; i += 32) s->sqrt_info[i] = Lm[i % 15][i / 15];  // transpose
}

// One CTA per (pre-integration slot, member): executes the member's jobs for that slot in list order (new
// IntegrationBase, push_back of the samples that arrived since the last solve: processIMU / slideWindow /
// repropagate, estimator.cpp:84-118, 1070-1081), then refreshes the cached sqrt_info if the slot takes part in
// this frame's problem.
__global__ void __launch_bounds__(256) preint_jobs_kernel(BaSeq* __restrict__ seqs) {
    __shared__ PreintSmem sm;
    __shared__ double sqA[15][31], sqL[15][15];
    const BaSeq& q = seqs[blockIdx.y];
    const int slot = blockIdx.x;
    const int nj = q.n_jobs;
    PreInt* pre = q.p.preint + slot;
    for (int j = 0; j < nj; j++) {
        const PreintJob& job = q.jobs[j];
        if (job.slot != slot) continue;  // CTA-uniform
        if (job.type == 0)
            preint_init_dev(pre, job);
        else if (job.n > 0)
            preint_push_dev(pre, job.n, q.samples + 7 * (size_t)job.sample_off, q.noise[0], q.noise[1], q.noise[2], q.noise[3], sm);
    }
    if ((q.sqrt_mask >> slot) & 1u) {
        __syncthreads();
        if (threadIdx.x < 32) sqrt_info_dev(pre, sqA, sqL);
    }
}

// ------------------------------------------------------------------------------------------------
// Copies a member's descriptor part into shared memory (kernel parameters used to carry it; with a batch it lives
// in device memory and every field would otherwise be a dependent global load).
template <class T>
__device__ __forceinline__ void load_desc(T* dst, const T* src) {
    static_assert(sizeof(T) % 8 == 0, "descriptor structs are multiples of 8 bytes");
    const int nth = blockDim.x * blockDim.y * blockDim.z;
    const int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
    for (int i = tid; i < (int)(sizeof(T) / 8); i += nth)
        reinterpret_cast<unsigned long long*>(dst)[i] = reinterpret_cast<const unsigned long long*>(src)[i];
    __syncthreads();
}

}  // namespace vb

#include "ba_assemble.cuh"
#include "chol_packed.cuh"

namespace vb {

// ------------------------------------------------------------------------------------------------
namespace {

__device__ __forceinline__ double block_sum(double v, double* red) {
    v = warp_sum_d(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0;
    for (unsigned w = 0; w < blockDim.x / 32; w++) s += red[w];
    return s;
}

// q = v^T H v over all parameters (H = [[Hfull, Hpl^T], [Hpl, diag(Hll)]], the landmark rows of Hpl in their sparse form)
__device__ double quad_form(const BaProblem& p, const BaAccum& a, const double* v, double* tmp, double* red) {
    const int D = p.dims.D, L = p.dims.L;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x / 32;
    double part = 0;
    for (int r = wid; r < D; r += nw) {
        double s = 0;
        for (int c = lane; c < D; c += 32) s += p.Hfull[(size_t)r * D + c] * v[c];
        s = warp_sum_d(s);
        if (lane == 0) part += v[r] * s;
    }
    for (int l = wid; l < L; l += nw) {
        const double s = lm_row_dot(p, a, l, v, lane);
        if (lane == 0) part += v[D + l] * (2.0 * s + a.lmW[(size_t)l * p.dims.lw + LW_HLL] * v[D + l]);
    }
    (void)tmp;
    return block_sum(part, red);
}

// cholesky_packed / chol_solve_packed and the CHOL_* constants: chol_packed.cuh (shared with pg_kernels.cu).

// Slow path: recompute S for a new mu inside the single step CTA (only after a failed factorisation): every entry of a
// pose-type block pair walks all landmarks in order.
__device__ void reduce_single_cta(const BaProblem& p, const BaAccum& a, double mu, int first) {
    const BaDims& d = p.dims;
    const int D = d.D, L = d.L, NV = num_vblocks(d);
    for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {  // S = Hfull everywhere first
        const int r = idx / D, c = idx % D;
        if (r > c) continue;
        const double h = p.Hfull[idx];
        p.S[idx] = h;
        p.S[(size_t)c * D + r] = h;
        p.Spk[(size_t)c * (c + 1) / 2 + r] = h;
    }
    for (int c = threadIdx.x; c < D; c += blockDim.x) p.gred[c] = a.gp[c];
    __syncthreads();
    // entries of the pose-type block pairs: 36 slots per pair
    for (int e = threadIdx.x; e < NV * NV * 36; e += blockDim.x) {
        const int pair = e / 36, t = e - 36 * pair;
        const int TA = pair / NV, TB = pair - TA * NV;
        if (TA > TB) continue;
        const VBlock A = vblock(d, TA), B = vblock(d, TB);
        const int i = t / B.dim, j = t - i * B.dim;
        if (t >= A.dim * B.dim || (TA == TB && i > j)) continue;
        double E = 0.0, gE = 0.0;
        for (int l = 0; l < L; l++) {
            const int rl = d.col_relo >= 0 ? p.lm_relo[l] : 0;
            const int an = p.lm_anchor[l], s0 = p.lm_start[l], nobs = p.lm_start[l + 1] - s0 - rl;
            if (!lm_covers(A, an, nobs, rl) || !lm_covers(B, an, nobs, rl)) continue;
            const double* rec = a.lmW + (size_t)l * d.lw;
            const double inv = lm_inv_lambda(p, a, l, mu, first);
            const double wa = lm_w(a, d.oj, rec, A, i, an, s0, nobs);
            E += wa * inv * lm_w(a, d.oj, rec, B, j, an, s0, nobs);
            if (TA == TB && i == j) gE += wa * inv * rec[LW_GL];
        }
        const int r = A.col + i, c = B.col + j;
        const double sv = p.Hfull[(size_t)r * D + c] - E;
        p.S[(size_t)r * D + c] = sv;
        p.S[(size_t)c * D + r] = sv;
        p.Spk[(size_t)c * (c + 1) / 2 + r] = sv;
        if (TA == TB && i == j) p.gred[r] = a.gp[r] - gE;
    }
    __syncthreads();
}

}  // namespace

// 1-D TMA bulk copy global -> shared (cp.async.bulk) completing on an mbarrier: the packed Schur complement
// (119 KB at the shipped sizes) lands in shared memory in one asynchronous transaction instead of 29 load/store round
// trips per thread (measured 15 k cycles per iteration for the loop).
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier generic-proxy accesses to dst are ordered first
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// The same transfer as `chunk`-byte pieces issued back to back by one thread: several bulk requests in flight drain a 119 KB
// matrix from L2 faster than one request walking it alone (17 k cycles measured for the single copy, harness/debug_backend.py).
__device__ __forceinline__ void bulk_g2s_chunked(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned chunk, unsigned long long* bar) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    for (unsigned off = 0; off < bytes; off += chunk) {
        const unsigned nb = bytes - off < chunk ? bytes - off : chunk;
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem) + off),
                     "l"((const char*)src_gmem + off), "r"(nb), "r"(smem_u32(bar))
                     : "memory");
    }
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// Generic-proxy stores of this thread to global memory are ordered before later async-proxy (bulk copy) reads of the same
// addresses.  Every thread that wrote Spk runs it before the barrier that precedes a bulk copy of Spk in the same kernel.
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// cp.async.bulk moves multiples of 16 bytes: an odd count is rounded up, the extra double lands on Lp[D (D + 1) / 2] (the first
// entry of the right-hand-side row, written after the transfer has completed; Spk has BA_SPK_SLACK behind the largest D)
__device__ __forceinline__ unsigned spk_copy_bytes(int D) { return (unsigned)((((D * (D + 1) / 2) + 1) & ~1) * sizeof(double)); }

// Loads the regularised reduced system of the step into the packed array Lp (D + 1 rows): p.Spk + mu E with
// E = p.diag^2 / p.scale^2 on the diagonal, and p.gred as row D (the right-hand side the factorisation carries along).
// bulk: Lp is in shared memory and arrives by the bulk copy completing on `bar`; copy_in_flight says the caller has issued
// that copy already (it is cleared here), otherwise it is issued here (a retry with a larger mu).  Without bulk, Lp (shared
// or global) is filled with plain loads.  Ends on a barrier.
__device__ __forceinline__ void step_load_system(const BaProblem& p, double* Lp, double mu, int D, bool bulk, bool& copy_in_flight,
                                                 unsigned long long* bar, unsigned& phase) {
    const int tid = threadIdx.x, nt = blockDim.x;
    if (bulk) {
        if (!copy_in_flight) {  // a retry with a larger mu: fetch the matrix again
            __syncthreads();    // every thread is done with the previous contents of Lp
            if (tid == 0) bulk_g2s_chunked(Lp, p.Spk, spk_copy_bytes(D), 8192u, bar);
        }
        copy_in_flight = false;
        const int npk = D * (D + 1) / 2;
        double rhs[2];  // row D: the right-hand side (D <= 2 nt), fetched while the transfer runs
#pragma unroll
        for (int u = 0; u < 2; u++) rhs[u] = tid + u * nt < D ? p.gred[tid + u * nt] : 0.0;
        mbar_wait(bar, phase);
        phase ^= 1;
#pragma unroll
        for (int u = 0; u < 2; u++)
            if (tid + u * nt <= D) Lp[npk + tid + u * nt] = rhs[u];
    } else {
        const int npk = D * (D + 1) / 2;
        for (int idx = tid; idx < npk; idx += nt) Lp[idx] = p.Spk[idx];
        for (int j = tid; j <= D; j += nt) Lp[npk + j] = j < D ? p.gred[j] : 0.0;  // row D: the right-hand side
    }
    __syncthreads();
    for (int i = tid; i < D; i += nt) {
        const double s_ = p.scale[i];
        Lp[(size_t)i * (i + 1) / 2 + i] += mu * (p.diag[i] * p.diag[i]) / (s_ * s_);
    }
    __syncthreads();
}

// After a successful cholesky_packed(Lp, ..., D, ..., D + 1): ysm = (S + mu E)^-1 gred.  Row D of Lp holds L^-1 gred already,
// so only the backward substitution is left.  Ends on a barrier.
__device__ __forceinline__ void step_solve(const double* Lp, const double* linv, int D, double* ysm) {
    const int npk = D * (D + 1) / 2;
    for (int j = threadIdx.x; j < D; j += blockDim.x) ysm[j] = Lp[npk + j];
    __syncthreads();
    chol_solve_packed(Lp, linv, D, ysm, false);
    __syncthreads();
}

__global__ void __launch_bounds__(512) ba_step_kernel(const BaSeq* __restrict__ seqs, int use_smem_chol) {
    extern __shared__ __align__(16) double chol_smem[];  // panel copy (CHOL_NB * CHOL_PS), then the packed factor
    __shared__ double red[32];
    __shared__ double rdiag[BA_MAX_D], ysm[BA_MAX_D], linv[(BA_MAX_D / CHOL_NB) * 64];
    __shared__ int flag;
    __shared__ BaProblem sp;
    const BaSeq& q = seqs[blockIdx.x];
    if (!q.active || q.st.done) return;
    load_desc(&sp, &q.p);
    const BaProblem& p = sp;
    SolverState* st = p.st;
    if (st->iteration >= st->max_iterations) {
        if (threadIdx.x == 0) st->done = 1;
        return;
    }
    const BaDims& d = p.dims;
    const int D = d.D, L = d.L, N = D + L;
    const int tid = threadIdx.x, nt = blockDim.x;
    __shared__ __align__(8) unsigned long long copy_bar;  // mbarrier of the bulk copy of the packed matrix
    unsigned copy_phase = 0;
    if (tid == 0) mbar_init(&copy_bar, 1);
    __syncthreads();
    const int lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    const int cur = st->cur;
    const BaAccum a = p.acc[cur];
    const BaWorkLayout wl = ba_work_layout(D, L);
    double* u = p.work + wl.u;          // Cauchy direction (unscaled variables)
    double* y = p.work + wl.y;          // Gauss-Newton solution
    double* delta = p.work + wl.delta;  // step in the original variables
    double* Lp = use_smem_chol ? chol_smem + CHOL_NB * CHOL_PS : p.work + wl.Lp;  // packed factor
    const int first = st->first;
    double mu = st->mu;
    bool linear_ok = true;
    long long c0 = clock64();
#define STAMP(k) do { if (tid == 0) { const long long c1_ = clock64(); st->clk[k] += c1_ - c0; c0 = c1_; } } while (0)
    const bool bulk_ok = use_smem_chol != 0;
    bool copy_in_flight = false;
    if (!st->reuse && bulk_ok) {
        // start the transfer of the packed Schur complement now: it overlaps the scaling / gradient phase below
        if (tid == 0) bulk_g2s_chunked(Lp, p.Spk, spk_copy_bytes(D), 8192u, &copy_bar);
        copy_in_flight = true;
    }
    if (!st->reuse) {
        for (int j = tid; j < N; j += nt) {
            const double hjj = j < D ? p.Hfull[(size_t)j * D + j] : a.lmW[(size_t)(j - D) * d.lw + LW_HLL];
            const double gj = j < D ? a.gp[j] : a.lmW[(size_t)(j - D) * d.lw + LW_GL];
            if (first) p.scale[j] = 1.0 / (1.0 + sqrt(hjj));
            const double s = p.scale[j];
            const double d2 = fmin(fmax(hjj * s * s, 1e-6), 1e32);
            const double dg = sqrt(d2);
            p.diag[j] = dg;
            p.grad[j] = gj * s / dg;
        }
        __syncthreads();
        STAMP(0);
        // regularised Gauss-Newton step: (S + mu E_p) y_p = gred, E = diag^2 / scale^2
        linear_ok = false;
        while (mu < 1.0) {
            step_load_system(p, Lp, mu, D, bulk_ok, copy_in_flight, &copy_bar, copy_phase);
            STAMP(2);
            const bool ok_ = cholesky_packed(Lp, chol_smem, D, rdiag, linv, &flag, D + 1);
            STAMP(3);
            if (ok_) {
                linear_ok = true;
                break;
            }
            mu *= 10.0;
            if (tid == 0) st->retries++;
            __syncthreads();
            if (mu < 1.0) {
                reduce_single_cta(p, a, mu, first);
                // the next attempt bulk-copies the Spk this CTA has just written with ordinary stores; the kernel boundary
                // that orders ba_reduce_kernel's stores before the first copy is missing here
                fence_proxy_async_global();
            }
        }
        if (copy_in_flight) {  // the loop did not run (mu already at its cap): drain the transfer before leaving
            mbar_wait(&copy_bar, copy_phase);
            copy_phase ^= 1;
            copy_in_flight = false;
        }
        if (linear_ok) {
            step_solve(Lp, linv, D, ysm);
            STAMP(4);
            for (int j = tid; j < D; j += nt) y[j] = ysm[j];
            // landmark back-substitution, 8 lanes per landmark (4 landmarks per warp in flight: the loop is bound by the
            // latency of the record reads, 25 k cycles per iteration with a warp per landmark)
            for (int l0 = 4 * wid; l0 < L; l0 += 4 * nw) {
                const int l = l0 + (lane >> 3);
                const double s = lm_row_dot8(p, a, l, L, ysm, lane & 7);
                if (l < L && (lane & 7) == 0) y[D + l] = (a.lmW[(size_t)l * d.lw + LW_GL] - s) * lm_inv_lambda(p, a, l, mu, first);
            }
            __syncthreads();
            for (int j = tid; j < N; j += nt) p.gn[j] = -p.diag[j] * y[j] / p.scale[j];
            STAMP(5);
        }
        if (tid == 0) {
            st->mu = mu;
            st->reuse = 1;
            st->first = 0;
            st->alpha_valid = 0;
        }
        __syncthreads();
    }
    // ---- traditional dogleg (DoglegStrategy::ComputeTraditionalDoglegStep)
    bool valid = false;
    double mcc = 0, dogleg_norm = 0;
    if (linear_ok) {
        double p1 = 0, p2 = 0, p3 = 0;
        for (int j = tid; j < N; j += nt) {
            p1 += p.grad[j] * p.grad[j];
            p2 += p.gn[j] * p.gn[j];
            p3 += p.grad[j] * p.gn[j];
        }
        const double gg = block_sum(p1, red), nn = block_sum(p2, red), gdn = block_sum(p3, red);
        const double gradient_norm = sqrt(gg), gn_norm = sqrt(nn);
        const double radius = st->radius;
        double ca = 0, cb = 0;  // step = ca * gradient + cb * gauss_newton  (trust-region-scaled space)
        if (gn_norm <= radius) {
            cb = 1.0;
            dogleg_norm = gn_norm;
        } else {
            // The Cauchy step length alpha = |g|^2 / |J D^-1 g|^2 needs one product with the full Hessian; it is
            // only evaluated when the Gauss-Newton step leaves the trust region (never at the default radius 1e4
            // unless steps were rejected).
            if (!st->alpha_valid) {
                for (int j = tid; j < N; j += nt) u[j] = p.grad[j] / p.diag[j] * p.scale[j];
                __syncthreads();
                const double uHu = quad_form(p, a, u, nullptr, red);
                if (tid == 0) {
                    st->alpha = gg / uHu;
                    st->alpha_valid = 1;
                }
                __syncthreads();
            }
            const double alpha = st->alpha;
            if (gradient_norm * alpha >= radius) {
                ca = -(radius / gradient_norm);
                dogleg_norm = radius;
            } else {
                const double b_dot_a = -alpha * gdn;
                const double a_sq = (alpha * gradient_norm) * (alpha * gradient_norm);
                const double bma = a_sq - 2 * b_dot_a + gn_norm * gn_norm;
                const double c = b_dot_a - a_sq;
                const double dd = sqrt(c * c + bma * (radius * radius - a_sq));
                const double beta = (c <= 0) ? (dd - c) / bma : (radius * radius - a_sq) / (dd + c);
                ca = -alpha * (1.0 - beta);
                cb = beta;
                dogleg_norm = -1.0;  // computed below
            }
        }
        double pn = 0, pg = 0, pe = 0;
        for (int j = tid; j < N; j += nt) {
            const double sd = ca * p.grad[j] + cb * p.gn[j];
            pn += sd * sd;
            const double s_ = p.scale[j];
            const double dl = sd / p.diag[j] * s_;  // undo trust-region diagonal and Jacobi scaling
            delta[j] = dl;
            pg += dl * (j < D ? a.gp[j] : a.lmW[(size_t)(j - D) * d.lw + LW_GL]);
            pe += dl * dl * (p.diag[j] * p.diag[j]) / (s_ * s_);
        }
        const double sn = block_sum(pn, red), dg = block_sum(pg, red), dEd = block_sum(pe, red);
        if (dogleg_norm < 0) dogleg_norm = sqrt(sn);
        double dHd;
        if (ca == 0.0 && cb == 1.0) {
            // full Gauss-Newton step: (H + mu E) delta = -g  =>  delta^T H delta = -delta^T g - mu delta^T E delta
            dHd = -dg - st->mu * dEd;
        } else {
            __syncthreads();
            dHd = quad_form(p, a, delta, nullptr, red);
        }
        mcc = -(dg + 0.5 * dHd);
        valid = mcc > 0.0;
        STAMP(6);
    }
    if (!valid) {  // HandleInvalidStep + DoglegStrategy::StepIsInvalid
        if (tid == 0) {
            st->iteration++;
            st->cand_valid = 0;
            st->invalid_streak++;
            if (st->invalid_streak >= 5) st->done = 4;
            st->mu = st->mu * 10.0;
            st->reuse = 0;
            if (st->iteration >= st->max_iterations && !st->done) st->done = 1;
        }
        return;
    }
    // ---- candidate point and the norms the tolerance tests need
    __syncthreads();
    const BaStates xc = p.x[cur], xn = p.x[1 - cur];
    double xs = 0, ss = 0;
    const int F = d.W + 1;
    for (int f = tid; f < F; f += nt) {
        double out[7];
        pose_plus(xc.pose + 7 * f, delta + 6 * f, out);
        for (int q = 0; q < 7; q++) {
            const double o = xc.pose[7 * f + q];
            xn.pose[7 * f + q] = out[q];
            xs += o * o;
            ss += (o - out[q]) * (o - out[q]);
        }
    }
    for (int i = tid; i < 9 * F; i += nt) {
        const double o = xc.sb[i], nv = o + delta[d.col_sb + i];
        xn.sb[i] = nv;
        xs += o * o;
        ss += (o - nv) * (o - nv);
    }
    if (tid == 0) {
        if (d.col_ex >= 0) {
            double out[7];
            pose_plus(xc.ex, delta + d.col_ex, out);
            for (int q = 0; q < 7; q++) {
                const double o = xc.ex[q];
                xn.ex[q] = out[q];
                xs += o * o;
                ss += (o - out[q]) * (o - out[q]);
            }
        } else
            for (int q = 0; q < 7; q++) xn.ex[q] = xc.ex[q];
        if (d.col_td >= 0) {
            const double o = xc.td[0], nv = o + delta[d.col_td];
            xn.td[0] = nv;
            xs += o * o;
            ss += (o - nv) * (o - nv);
        } else
            xn.td[0] = xc.td[0];
    }
    if (tid == 32 && d.col_relo >= 0) {  // relo_Pose: one more PoseLocalParameterization block
        double out[7];
        pose_plus(xc.relo, delta + d.col_relo, out);
        for (int q = 0; q < 7; q++) {
            const double o = xc.relo[q];
            xn.relo[q] = out[q];
            xs += o * o;
            ss += (o - out[q]) * (o - out[q]);
        }
    }
    for (int l = tid; l < L; l += nt) {
        const double o = xc.lam[l], nv = o + delta[D + l];
        xn.lam[l] = nv;
        xs += o * o;
        ss += (o - nv) * (o - nv);
    }
    const double x_norm2 = block_sum(xs, red), step_norm2 = block_sum(ss, red);
    STAMP(7);
    if (tid == 0) {
        st->iteration++;
        st->cand_valid = 1;
        st->invalid_streak = 0;
        st->model_cost_change = mcc;
        st->dogleg_step_norm = dogleg_norm;
        st->x_norm = sqrt(x_norm2);
        st->step_norm = sqrt(step_norm2);
    }
}

// ------------------------------------------------------------------------------------------------
// Marginalisation.  Column layout of the dense system: [m_dense | m_landmarks (diagonal block) | kept n].
// MarginalizationInfo::preMarginalize + the assembly part of marginalize (marginalization_factor.cpp:110-172): the factors
// that touch the dropped blocks are evaluated at the re-anchored point x[0] into their records (marg_eval_kernel, the
// same device code as the solve's linearisation, with the extrinsic block always live: it is a parameter of the prior even
// when the solve keeps it constant), then the dense system is gathered entry by entry in a fixed order (marg_gather_kernel).
constexpr int MARG_OJ = OJ_FULL, MARG_LW = LW_FULL;
constexpr int MARG_QMAX = BA_MARG_MAX_DENSE + 1 + BA_MAX_PRIOR_N;  // non-landmark columns: m_dense + kept, and one spare

// Clears the members' marginalisation systems (Am P x P, bm P).
__global__ void __launch_bounds__(256) marg_zero_kernel(const BaSeq* __restrict__ seqs) {
    const BaSeq& q = seqs[blockIdx.y];
    if (!q.active || !q.do_marg) return;
    const size_t P = (size_t)q.mp.P, total = P * P + P;
    double* Am = q.mp.Am;
    double* bm = q.mp.bm;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        if (i < P * P) Am[i] = 0.0;
        else bm[i - P * P] = 0.0;
    }
}

template <bool TD>
__global__ void __launch_bounds__(32 * LIN_WARPS) marg_eval_kernel(const BaSeq* __restrict__ seqs) {
    __shared__ double sJraw[450], srr[16];
    __shared__ double sdx[BA_MAX_PRIOR_N], sred[BA_MAX_PRIOR_N];
    __shared__ BaProblem sp;
    const BaSeq& q = seqs[blockIdx.y];
    if (!q.active || !q.do_marg) return;
    const int n_lm = q.mp.n_lm, nb_vis = (n_lm + LIN_WARPS - 1) / LIN_WARPS;
    if ((int)blockIdx.x >= nb_vis + 2) return;
    load_desc(&sp, &q.p);
    const BaProblem& p = sp;
    const BaStates x = p.x[0];
    const BaAccum a = p.acc[0];  // the solve is over: its records are free
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int blk = blockIdx.x;
    if (blk < nb_vis) {
        const int li = blk * LIN_WARPS + wid;
        if (li < n_lm) lin_visual<true, TD>(p, x, a, MARG_OJ, MARG_LW, q.mp.lms[li], lane, false);
    } else if (blk == nb_vis) {
        if (q.mp.use_imu) lin_imu(p, x, a, 0, sJraw, srr);
    } else {
        lin_prior(p, x, a, sdx, sred);
    }
}

struct MargCol {  // a non-landmark column of the marginalisation system
    short type, frame, i;  // 0 pose, 1 speed-bias, 2 ex, 3 td
};

__global__ void __launch_bounds__(128) marg_gather_kernel(const BaSeq* __restrict__ seqs, int dense_ctas) {
    __shared__ BaProblem sp;
    __shared__ MargPlan smp;
    __shared__ MargCol mcol[MARG_QMAX];
    __shared__ short mfull[MARG_QMAX];  // reduced index -> column in Am
    __shared__ short pinv_m[MARG_QMAX]; // reduced index -> row of the previous prior, or -1
    const BaSeq& q = seqs[blockIdx.y];
    if (!q.active || !q.do_marg) return;
    load_desc(&sp, &q.p);
    load_desc(&smp, &q.mp);
    const BaProblem& p = sp;
    const MargPlan& mp = smp;
    const BaDims& d = p.dims;
    const BaAccum a = p.acc[0];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int md = mp.m_dense, nl = mp.n_lm, n = mp.n, P = mp.P, Q = md + n;
    const int F = d.W + 1;
    // reduced (non-landmark) columns: decode through the plan's column tables
    for (int k = tid; k < Q; k += nt) {
        mfull[k] = (short)(k < md ? k : k + nl);
        pinv_m[k] = -1;
    }
    __syncthreads();
    auto reduced = [&](int col) { return col < md ? col : col - nl; };
    for (int f = tid; f < F; f += nt) {
        if (mp.col_pose[f] >= 0)
            for (int i = 0; i < 6; i++) mcol[reduced(mp.col_pose[f] + i)] = MargCol{0, (short)f, (short)i};
        if (mp.col_sb[f] >= 0)
            for (int i = 0; i < 9; i++) mcol[reduced(mp.col_sb[f] + i)] = MargCol{1, (short)f, (short)i};
    }
    if (tid == 0) {
        if (mp.col_ex >= 0)
            for (int i = 0; i < 6; i++) mcol[reduced(mp.col_ex + i)] = MargCol{2, 0, (short)i};
        if (mp.col_td >= 0) mcol[reduced(mp.col_td)] = MargCol{3, 0, 0};
    }
    for (int b = tid; b < p.prior.nblocks; b += nt) {
        const int type = p.prior.type[b], idx = p.prior.index[b], off = p.prior.off[b];
        const int base = type == 0 ? mp.col_pose[idx] : type == 1 ? mp.col_sb[idx] : type == 2 ? mp.col_ex : mp.col_td;
        const int sz = type == 0 || type == 2 ? 6 : type == 1 ? 9 : 1;
        for (int i = 0; i < sz; i++) pinv_m[reduced(base + i)] = (short)(off + i);
    }
    __syncthreads();
    const int blk = blockIdx.x;
    if (blk >= dense_ctas) {
        // landmark columns: one warp per marginalised landmark writes its column, diagonal and right-hand side
        const int li = (blk - dense_ctas) * (nt / 32) + (tid >> 5), lane = tid & 31;
        if (li >= nl) return;
        const int l = mp.lms[li], cl = mp.col_lm[li];
        // (a relocalisation match behind the track is not part of the marginalisation)
        const int an = p.lm_anchor[l], s0 = p.lm_start[l], nobs = p.lm_start[l + 1] - s0 - (d.col_relo >= 0 ? p.lm_relo[l] : 0);
        const double* rec = a.lmW + (size_t)l * MARG_LW;
        for (int idx = lane; idx < 6 * (nobs + 1); idx += 32) {
            const int t = idx / 6, i = idx - 6 * t;
            const double w = t == 0 ? rec[LW_WI + i] : a.obsJ[(size_t)(s0 + t - 1) * MARG_OJ + OJ_WJ + i];
            const int col = mp.col_pose[an + t] + i;
            if (col < cl) mp.Am[(size_t)col * P + cl] = w;
            else mp.Am[(size_t)cl * P + col] = w;
        }
        if (lane < 6) {
            const int col = mp.col_ex + lane;
            mp.Am[(size_t)cl * P + col] = rec[LW_WE + lane];  // kept columns come after the landmark columns
        }
        if (lane == 6 && d.est_td && mp.col_td >= 0) mp.Am[(size_t)cl * P + mp.col_td] = rec[LW_WT];
        if (lane == 7) {
            mp.Am[(size_t)cl * P + cl] = rec[LW_HLL];
            mp.bm[cl] = rec[LW_GL];
        }
        return;
    }
    // dense part: upper-triangle entries between non-landmark columns
    const int total = Q * (Q + 1) / 2;
    for (int idx = blk * nt + tid; idx < total; idx += dense_ctas * nt) {
        int cb = (int)((sqrtf(8.f * (float)idx + 1.f) - 1.f) * 0.5f);
        while (cb * (cb + 1) / 2 > idx) cb--;
        while ((cb + 1) * (cb + 2) / 2 <= idx) cb++;
        const int ra = idx - cb * (cb + 1) / 2;  // ra <= cb, reduced indices
        const MargCol A = mcol[ra], B = mcol[cb];
        // previous prior (J^T J = A), in the order the prior rows map to the columns
        double h = 0.0;
        if (p.prior.n > 0 && pinv_m[ra] >= 0 && pinv_m[cb] >= 0) h = p.prior.A[(size_t)pinv_m[ra] * p.prior.n + pinv_m[cb]];
        // IMU factor between frames 0 and 1
        auto loc0 = [](const MargCol& c) { return c.type > 1 || c.frame > 1 ? -1 : (c.frame == 0 ? (c.type == 0 ? c.i : 6 + c.i) : (c.type == 0 ? 15 + c.i : 21 + c.i)); };
        const double* irec = a.imuJ;
        if (mp.use_imu && irec[IMUJ_VALID] != 0.0) {
            const int la = loc0(A), lb = loc0(B);
            if (la >= 0 && lb >= 0) {
                double s = 0;
                for (int k = 0; k < 15; k++) s += irec[IMUJ_JW + k * 30 + la] * irec[IMUJ_JW + k * 30 + lb];
                h += s;
            }
        }
        // visual factors of the marginalised landmarks (all anchored in the dropped frame)
        const bool va = A.type != 1, vb_ = B.type != 1;
        double g = 0.0;
        if (va && vb_) {
            VBlock VA{A.type, A.frame, 0, A.type == 3 ? 1 : 6}, VB{B.type, B.frame, 0, B.type == 3 ? 1 : 6};
            // block order pose < ex < td with poses by frame: (ra <= cb) does not imply it, so order the pair explicitly
            const bool swap = (VA.type > VB.type) || (VA.type == 0 && VB.type == 0 && VA.frame > VB.frame);
            for (int li = 0; li < nl; li++) {
                const int l = mp.lms[li];
                const int an = p.lm_anchor[l], s0 = p.lm_start[l], nobs = p.lm_start[l + 1] - s0 - (d.col_relo >= 0 ? p.lm_relo[l] : 0);
                if (!lm_covers(VA, an, nobs, 0) || !lm_covers(VB, an, nobs, 0)) continue;
                const double* rec = a.lmW + (size_t)l * MARG_LW;
                h += swap ? vis_entry(a, MARG_OJ, rec, VB, VA, B.i, A.i, an, s0, nobs) : vis_entry(a, MARG_OJ, rec, VA, VB, A.i, B.i, an, s0, nobs);
                if (ra == cb) g += vis_grad(a, MARG_OJ, rec, VA, A.i, an, s0, nobs);
            }
        }
        const int fa = mfull[ra], fb = mfull[cb];
        if (fa <= fb) mp.Am[(size_t)fa * P + fb] = h;
        else mp.Am[(size_t)fb * P + fa] = h;
        if (ra == cb) {
            double gb = g;
            if (p.prior.n > 0 && pinv_m[ra] >= 0) gb += a.gpr[pinv_m[ra]];
            if (mp.use_imu && irec[IMUJ_VALID] != 0.0) {
                const int la = loc0(A);
                if (la >= 0) {
                    double s = 0;
                    for (int k = 0; k < 15; k++) s += irec[IMUJ_JW + k * 30 + la] * irec[IMUJ_RW + k];
                    gb += s;
                }
            }
            mp.bm[fa] = gb;
        }
    }
}

constexpr int MARG_THREADS = 512;

// landmark rows marg_solve_kernel stages per round: 8 when the reduced system lives in global memory (the large windows:
// with 16, the scratch of the window of 22 frames with extrinsic and td, n = 148, overflows the 227 KB of an H100 CTA)
__host__ __device__ inline int marg_stage_rows(bool w_in_global) { return w_in_global ? 8 : 16; }

// doubles of the scratch area Ev: staged landmark rows (2 x marg_stage_rows x qp) or the n x md products Y and X
// (+ a copy of the scaled eigenvectors, n x (n|1), when the reduced system lives in shared memory, i.e. small windows)
__host__ __device__ inline int marg_scratch_doubles(int md, int n, bool w_in_global) {
    const int q = md + n, qp = (q + 3) & ~3, ldm = md + (md & 1);
    int a = 2 * marg_stage_rows(w_in_global) * qp;
    const int b = n * (ldm + md), c = w_in_global ? 0 : n * (n | 1);
    a = a > b ? a : b;
    a = a > c ? a : c;
    if (!w_in_global) {  // Wk | Ev together hold the work arrays of the prior's eps floor (prior_floor.h) once both are dead
        const int f = prior_floor_work(n, MARG_THREADS, 32) - ((q * q + 1) & ~1);
        a = a > f ? a : f;
    }
    return (a + 1) & ~1;
}

// Single CTA.  Dynamic shared memory: Wk (q x q), Ev (scratch), Vv ((ldx+1)^2: matrix in / eigenvectors out), bw (q), tv.
// Both eigen-decompositions (the dense marginalised block T and the new prior A') use the tridiagonal-QL solver of
// sym_eig.h: eigenvector k is the COLUMN k of Vv (odd leading dimension: conflict-free row walks).
__global__ void __launch_bounds__(MARG_THREADS) marg_solve_kernel(const BaSeq* __restrict__ seqs, double eps) {
    extern __shared__ __align__(16) double sm[];
    __shared__ double red[32];
    __shared__ double dval[BA_MAX_PRIOR_N], ework[BA_MAX_PRIOR_N], cs[4 * BA_MAX_PRIOR_N], scal[16];
    __shared__ MargPlan smp;
    {
        const BaSeq& q = seqs[blockIdx.x];
        if (!q.active || !q.do_marg) return;
        load_desc(&smp, &q.mp);
    }
    const MargPlan& mp = smp;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int md = mp.m_dense, nl = mp.n_lm, n = mp.n, P = mp.P;
    const int q = md + n;
    const int ldm = md + (md & 1), ldn = n + (n & 1), ldx = max(ldm, ldn);
    const int esz = marg_scratch_doubles(md, n, mp.w_in_global != 0);
    // the reduced system W (q x q) lives in shared memory when it fits (the shipped window), else in global memory
    double* Wk = mp.w_in_global ? mp.Wglobal : sm;
    double* Ev = mp.w_in_global ? sm : sm + ((q * q + 1) & ~1);  // esz, 16-byte aligned (128-bit loads of the staged rows)
    double* Vv = Ev + esz;            // (ldx+1)^2
    double* bw = Vv + (ldx + 1) * (ldx + 1);  // q
    double* tv = bw + q;              // ldx
    auto symA = [&](int a, int b) { return a <= b ? mp.Am[(size_t)a * P + b] : mp.Am[(size_t)b * P + a]; };
    auto full = [&](int a) { return a < md ? a : a + nl; };  // index in Am of reduced index a
    long long mclk[6] = {0, 0, 0, 0, 0, 0};
    long long mc0 = clock64();
#define MSTAMP(k) do { const long long c1_ = clock64(); mclk[k] = c1_ - mc0; mc0 = c1_; } while (0)
    // 1. eliminate the landmark columns (exactly diagonal block): W -= sum_c w_c w_c^T / d_c over the landmarks c.
    //    Register-tiled: a thread owns one 4x4 tile of the upper triangle of W (q = 90 -> 276 tiles) and accumulates
    //    over ALL landmarks in registers; the landmark rows are staged MCH at a time in shared memory (raw and scaled by
    //    1/d_c, row stride qp = q rounded up to 4 so that a tile operand is two 128-bit loads).  Landmark rows are sparse
    //    (only the observing frames' pose blocks): a tile skips a landmark whose scaled operand is zero.
    const int qp = (q + 3) & ~3, nt4 = qp >> 2, ntile = nt4 * (nt4 + 1) / 2;
    const int MCH = marg_stage_rows(mp.w_in_global != 0);  // the order of the sums does not depend on it
    double* Wl = Ev;             // MCH x qp raw rows
    double* Ws = Ev + MCH * qp;  // MCH x qp rows scaled by 1 / d_c (0 when d_c <= eps)
    double* invd = tv;           // MCH: 1 / d_c, then b_c in invd + MCH
    const int tile_threads = nt - q;  // the last q threads accumulate the right-hand side (first round only)
    for (int t0 = 0; t0 < ntile; t0 += tile_threads) {  // one round at the shipped sizes; more for larger windows
        const int tile = t0 + tid;
        const bool has_tile = tid < tile_threads && tile < ntile;
        const bool has_rhs = t0 == 0 && tid >= tile_threads;
        int ta = 0, tb = 0;
        if (has_tile) {  // tile index -> (ta <= tb): row ta holds tiles tb = ta .. nt4-1
            int rem = tile;
            while (rem >= nt4 - ta) {
                rem -= nt4 - ta;
                ta++;
            }
            tb = ta + rem;
        }
        double acc[4][4];
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int c = 0; c < 4; c++) acc[r][c] = 0.0;
        double bacc = 0.0;  // sum_c w_c[aa] b_c / d_c
        for (int c0 = 0; c0 < nl; c0 += MCH) {
            const int cn = min(MCH, nl - c0);
            if (tid < cn) {
                const int fc = md + c0 + tid;
                const double dc = mp.Am[(size_t)fc * P + fc];
                invd[tid] = dc > eps ? 1.0 / dc : 0.0;
                invd[MCH + tid] = mp.bm[fc];
            }
            __syncthreads();
            for (int idx = tid; idx < MCH * qp; idx += nt) {
                const int c = idx / qp, aa = idx - c * qp;
                double v = 0.0;
                if (c < cn && aa < q) {
                    const int fc = md + c0 + c;
                    v = aa < md ? mp.Am[(size_t)aa * P + fc] : mp.Am[(size_t)fc * P + aa + nl];
                }
                Wl[idx] = v;
                Ws[idx] = c < cn ? v * invd[c] : 0.0;
            }
            __syncthreads();
            if (has_tile) {
                for (int c = 0; c < cn; c++) {
                    const double2* pa = reinterpret_cast<const double2*>(Ws + c * qp + 4 * ta);
                    const double2 a01 = pa[0], a23 = pa[1];
                    if (a01.x == 0.0 && a01.y == 0.0 && a23.x == 0.0 && a23.y == 0.0) continue;
                    const double2* pb = reinterpret_cast<const double2*>(Wl + c * qp + 4 * tb);
                    const double2 b01 = pb[0], b23 = pb[1];
                    const double av[4] = {a01.x, a01.y, a23.x, a23.y}, bv[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
                    for (int r = 0; r < 4; r++)
#pragma unroll
                        for (int cc = 0; cc < 4; cc++) acc[r][cc] += av[r] * bv[cc];
                }
            } else if (has_rhs) {
                const int aa = tid - tile_threads;
                for (int c = 0; c < cn; c++) bacc += Ws[c * qp + aa] * invd[MCH + c];
            }
            __syncthreads();
        }
        if (has_tile) {
#pragma unroll
            for (int r = 0; r < 4; r++)
#pragma unroll
                for (int cc = 0; cc < 4; cc++) {
                    const int aa = 4 * ta + r, bb = 4 * tb + cc;
                    if (aa <= bb && bb < q) {
                        const double v = symA(full(aa), full(bb)) - acc[r][cc];
                        Wk[aa * q + bb] = v;
                        Wk[bb * q + aa] = v;
                    }
                }
        } else if (has_rhs) {
            const int aa = tid - tile_threads;
            bw[aa] = mp.bm[full(aa)] - bacc;
        }
    }
    __syncthreads();
    // 2. pseudo-inverse of the dense marginalised block T (md x md, md <= 15).  The reference takes V diag(1/w where w > eps) V^T
    //    (marginalization_factor.cpp:268-275); whenever T - s I still has a Cholesky factor (s = max(2 eps, 64 ulp trace T):
    //    every eigenvalue beyond doubt above the floor) that is the plain inverse, computed by warp 0 from the factor of T:
    //    20 k cycles against 116 k for the decomposition.  Otherwise the decomposition decides pair by pair.
    const int ldvm = md | 1, ldvn = n | 1;
    __shared__ double Tl[16][17], Tinv[16][17];
    __shared__ int t_pd;
    MSTAMP(0);
    if (tid < 32) {
        const int lane = tid;
        double tr = 0.0;
        if (lane < md) tr = Wk[lane * q + lane];
        tr = warp_sum_d(tr);
        const double shift = fmax(2.0 * eps, 64.0 * 2.220446049250313e-16 * tr);
        bool ok = true;
        for (int pass = 0; pass < 2 && ok; pass++) {  // pass 0: T - shift I (the test), pass 1: T
            for (int idx = lane; idx < md * md; idx += 32) {
                const int i = idx / md, j = idx - i * md;
                Tl[i][j] = Wk[i * q + j] - ((i == j && pass == 0) ? shift : 0.0);
            }
            __syncwarp();
            for (int j = 0; j < md; j++) {  // lane i owns row i
                const double piv = Tl[j][j];
                if (!(piv > 0.0) || !(piv < 1e300)) {
                    ok = false;
                    break;
                }
                const double r = rsqrt(piv);
                double lij = 0.0;
                if (lane >= j && lane < md) {
                    lij = lane == j ? piv * r : Tl[lane][j] * r;
                    Tl[lane][j] = lij;
                }
                __syncwarp();
                if (lane > j && lane < md)
                    for (int c = j + 1; c <= lane; c++) Tl[lane][c] -= lij * Tl[c][j];
                __syncwarp();
            }
        }
        if (ok && lane < md) {  // column `lane` of T^-1: L z = e_lane, L^T x = z
            double x[16];
#pragma unroll
            for (int i = 0; i < 16; i++) {
                double v = i == lane ? 1.0 : 0.0;
                if (i < md) {
#pragma unroll
                    for (int c = 0; c < 16; c++)
                        if (c < i) v -= Tl[i][c] * x[c];
                    v /= Tl[i][i];
                }
                x[i] = i < md ? v : 0.0;
            }
#pragma unroll
            for (int i = 15; i >= 0; i--) {
                if (i < md) {
                    double v = x[i];
#pragma unroll
                    for (int c = 0; c < 16; c++)
                        if (c > i && c < md) v -= Tl[c][i] * x[c];
                    x[i] = v / Tl[i][i];
                }
            }
#pragma unroll
            for (int i = 0; i < 16; i++)
                if (i < md) Tinv[i][lane] = x[i];
        }
        if (lane == 0) t_pd = ok ? 1 : 0;
    }
    __syncthreads();
    double* X = Ev + (size_t)n * md;  // n x md
    if (t_pd) {
        MSTAMP(1);
        // 3. X = Wrm Tinv (n x md)
        for (int idx = tid; idx < n * md; idx += nt) {
            const int i = idx / md, j = idx - i * md;
            double s = 0;
            for (int k = 0; k < md; k++) s += Wk[(md + i) * q + k] * Tinv[k][j];
            X[idx] = s;
        }
        __syncthreads();
    } else {
        for (int idx = tid; idx < md * md; idx += nt) {
            const int i = idx / md, j = idx - i * md;
            Vv[i * ldvm + j] = Wk[i * q + j];
        }
        __syncthreads();
        sym_eig<CtaCtx, 3>(CtaCtx(), Vv, md, ldvm, dval, ework, cs, scal);  // md <= 15
        MSTAMP(1);
        for (int k = tid; k < md; k += nt) tv[k] = dval[k] > eps ? 1.0 / dval[k] : 0.0;
        __syncthreads();
        // 3. X = Wrm Tinv (n x md) computed directly from the eigen-factors: X = (Wrm V) diag(tv) V^T
        //    Y = Wrm V diag(tv) -> Ev as n x md
        for (int idx = tid; idx < n * md; idx += nt) {
            const int i = idx / md, k = idx - i * md;
            double s = 0;
            for (int j = 0; j < md; j++) s += Wk[(md + i) * q + j] * Vv[j * ldvm + k];
            Ev[idx] = s * tv[k];
        }
        __syncthreads();
        for (int idx = tid; idx < n * md; idx += nt) {
            const int i = idx / md, j = idx - i * md;
            double s = 0;
            for (int k = 0; k < md; k++) s += Ev[i * md + k] * Vv[j * ldvm + k];
            X[idx] = s;
        }
        __syncthreads();
    }
    double* Ap = mp.Aout;  // n x n (global, becomes the prior's A after thresholding)
    for (int idx = tid; idx < n * n; idx += nt) {
        const int i = idx / n, j = idx % n;
        double s = Wk[(md + i) * q + md + j];
        for (int k = 0; k < md; k++) s -= X[i * md + k] * Wk[k * q + md + j];
        Ap[idx] = s;
    }
    for (int i = tid; i < n; i += nt) {
        double s = bw[md + i];
        for (int k = 0; k < md; k++) s -= X[i * md + k] * bw[k];
        mp.gout[i] = s;
    }
    __syncthreads();
    if (mp.Araw)
        for (int idx = tid; idx < n * n; idx += nt) mp.Araw[idx] = 0.5 * (Ap[idx] + Ap[(idx % n) * n + idx / n]);
    if (mp.graw)
        for (int i = tid; i < n; i += nt) mp.graw[i] = mp.gout[i];
    // 4. the eps floor of A' (prior_floor.h): A+ = V S+ V^T, g0 = V 1+ V^T b', c0 = b'^T V S+^-1 V^T b'.  Only the eigenpairs at the
    //    noise floor are separated explicitly when the scratch behind Wk | Ev (both dead by now) holds the work arrays;
    //    otherwise (reduced system in global memory: the large windows) the full decomposition runs.
    __syncthreads();
    MSTAMP(2);
    __shared__ int fstats[2];
    {
        const int avail = (int)(Vv - sm);  // doubles in front of Vv
        double* fwork = (!mp.w_in_global && prior_floor_work(n, nt, 32) <= avail) ? sm : nullptr;
        double* fev = mp.w_in_global ? nullptr : Ev;
        if (n <= 96)
            prior_floor<CtaCtx, 3>(CtaCtx(), Ap, mp.gout, mp.cout, n, eps, Vv, ldvn, dval, ework, cs, scal, tv, fwork, fev, fstats);
        else
            prior_floor<CtaCtx, SE_PER_LANE_MAX>(CtaCtx(), Ap, mp.gout, mp.cout, n, eps, Vv, ldvn, dval, ework, cs, scal, tv, fwork, fev, fstats);
    }
    MSTAMP(3);
    if (tid == 0 && mp.graw) {  // the BA_MARG_DIAG diagnostics behind the n used entries
        double* diag = mp.graw + n;
        diag[0] = scal[4];              // A' decomposition: tridiagonalisation cycles
        diag[1] = (double)fstats[0];  // eigenpairs separated explicitly (-1: full decomposition)
        MSTAMP(4);
        for (int k = 0; k < BA_MARG_DIAG - 2; k++) diag[2 + k] = (double)mclk[k];
    }
}

size_t marg_solve_smem_bytes(int m_dense, int n, bool w_in_global) {
    const int q = m_dense + n;
    const int ldm = m_dense + (m_dense & 1), ldn = n + (n & 1), ldx = ldm > ldn ? ldm : ldn;
    const size_t esz = (size_t)marg_scratch_doubles(m_dense, n, w_in_global);
    return sizeof(double) * ((w_in_global ? 0 : (size_t)q * q + 1) + esz + (size_t)(ldx + 1) * (ldx + 1) + q + std::max(ldx, 32));
}

// ------------------------------------------------------------------------------------------------
// Estimator::double2vector (estimator.cpp:530-619) followed by vector2double (:486-528) on the device, one CTA per
// member: the solved window is re-anchored to the yaw and position of frame 0 before the solve (the 4 unobservable
// degrees of freedom), written to the member's output block for the host (Ps, Rs, Vs, Bas, Bgs, tic, ric, td, depths)
// and packed again into x[0], the linearisation point of this frame's marginalisation; the new prior's x0 is taken from it.
__global__ void __launch_bounds__(128) ba_finish_kernel(BaSeq* __restrict__ seqs) {
    __shared__ double sin_[ba_states_layout(BA_MAX_FRAMES, 0).lam];  // pose | sb | ex | td of x[cur] (the states layout)
    __shared__ double rot[9];
    BaSeq& q = seqs[blockIdx.x];
    if (!q.active) return;
    const BaProblem& p = q.p;
    const FinishPlan& fp = q.fin;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int F = p.dims.W + 1, L = p.dims.L;
    const int cur = q.st.cur;
    const BaStates xs = p.x[cur], xd = p.x[0];
    const BaStates sx = states_view(sin_, F, 0);
    for (int i = tid; i < 7 * F; i += nt) sx.pose[i] = xs.pose[i];
    for (int i = tid; i < 9 * F; i += nt) sx.sb[i] = xs.sb[i];
    for (int i = tid; i < 7; i += nt) sx.ex[i] = xs.ex[i];
    if (tid == 0) sx.td[0] = xs.td[0];
    __syncthreads();
    if (tid == 0) {
        const Mat3 R00 = qR(q_from_param(sx.pose));
        const Vec3 o0 = Vec3(fp.origin_ypr[0], fp.origin_ypr[1], fp.origin_ypr[2]);
        const Vec3 o00 = R2ypr(R00);
        const double y_diff = o0.x - o00.x;
        Mat3 rd = ypr2R(Vec3(y_diff, 0.0, 0.0));
        if (fabs(fabs(o0.y) - 90) < 1.0 || fabs(fabs(o00.y) - 90) < 1.0) {
            Mat3 R0;
            for (int k = 0; k < 9; k++) R0.m[k] = fp.Rs0[k];
            rd = mmul(R0, mT(R00));
        }
        for (int k = 0; k < 9; k++) rot[k] = rd.m[k];
    }
    __syncthreads();
    double* out = fp.out;
    {  // header: the final trust-region state
        const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&q.st);
        for (int i = tid; i < (int)(sizeof(SolverState) / 8); i += nt) reinterpret_cast<unsigned long long*>(out)[i] = src[i];
    }
    const BaOutLayout ol = ba_out_layout(F, L, p.dims.col_relo >= 0);
    Mat3 rd;
    for (int k = 0; k < 9; k++) rd.m[k] = rot[k];
    for (int f = tid; f < F; f += nt) {
        const double* pp = sx.pose + 7 * f;
        const double* sbp = sx.sb + 9 * f;
        const Mat3 R = mmul(rd, qR(qnormalized(q_from_param(pp))));
        const Vec3 P = mv(rd, Vec3(pp[0] - sx.pose[0], pp[1] - sx.pose[1], pp[2] - sx.pose[2])) + Vec3(fp.origin_P0[0], fp.origin_P0[1], fp.origin_P0[2]);
        const Vec3 V = mv(rd, Vec3(sbp[0], sbp[1], sbp[2]));
        double* o = out + ol.frames + BA_OUT_FRAME * f;
        o[0] = P.x; o[1] = P.y; o[2] = P.z;
        for (int k = 0; k < 9; k++) o[3 + k] = R.m[k];
        o[12] = V.x; o[13] = V.y; o[14] = V.z;
        for (int k = 0; k < 6; k++) o[15 + k] = sbp[3 + k];
        // vector2double
        const Quat qq = Quat::FromR(R);
        double* dp = xd.pose + 7 * f;
        dp[0] = P.x; dp[1] = P.y; dp[2] = P.z; dp[3] = qq.x; dp[4] = qq.y; dp[5] = qq.z; dp[6] = qq.w;
        double* ds = xd.sb + 9 * f;
        ds[0] = V.x; ds[1] = V.y; ds[2] = V.z;
        for (int k = 0; k < 6; k++) ds[3 + k] = sbp[3 + k];
    }
    if (tid == nt - 1) {
        const double* xe = sx.ex;
        const Mat3 ric = qR(q_from_param(xe));
        double* o = out + ol.ex;
        o[0] = xe[0]; o[1] = xe[1]; o[2] = xe[2];
        for (int k = 0; k < 9; k++) o[3 + k] = ric.m[k];
        o[12] = sx.td[0];
        const Quat qq = Quat::FromR(ric);
        xd.ex[0] = xe[0]; xd.ex[1] = xe[1]; xd.ex[2] = xe[2];
        xd.ex[3] = qq.x; xd.ex[4] = qq.y; xd.ex[5] = qq.z; xd.ex[6] = qq.w;
        xd.td[0] = sx.td[0];
    }
    if (tid == nt - 2 && p.dims.col_relo >= 0) {  // relo_r / relo_t of double2vector (estimator.cpp:598-605)
        const double* rp = xs.relo;
        const Mat3 Rr = mmul(rd, qR(qnormalized(q_from_param(rp))));
        const Vec3 Pr = mv(rd, Vec3(rp[0] - sx.pose[0], rp[1] - sx.pose[1], rp[2] - sx.pose[2])) + Vec3(fp.origin_P0[0], fp.origin_P0[1], fp.origin_P0[2]);
        double* o = out + ol.relo;
        for (int k = 0; k < 9; k++) o[k] = Rr.m[k];
        o[9] = Pr.x; o[10] = Pr.y; o[11] = Pr.z;
    }
    double* od = out + ol.depths;
    for (int l = tid; l < L; l += nt) {  // FeatureManager::setDepth, then getDepthVector
        const double dep = 1.0 / xs.lam[l];
        od[l] = dep;
        xd.lam[l] = 1. / dep;
    }
    __syncthreads();
    // linearisation point of the new prior: the packed values of the kept blocks (marginalization_factor.cpp:299-319)
    if (q.do_marg)
        for (int b = tid; b < fp.n_kept; b += nt) {
            const int type = fp.kept_type[b], idx = fp.kept_index[b];
            double* dst = fp.x0_out + 9 * b;
            const double* src = type == 0 ? xd.pose + 7 * idx : type == 1 ? xd.sb + 9 * idx : type == 2 ? xd.ex : xd.td;
            const int n = type == 0 || type == 2 ? 7 : type == 1 ? 9 : 1;
            for (int k = 0; k < 9; k++) dst[k] = k < n ? src[k] : 0.0;
        }
}

// ------------------------------------------------------------------------------------------------
// Single-factor evaluation for the parity tests (ve_debug_*): the device functions the solve uses, one thread.
__global__ void debug_visual_kernel(BaDims d, const double* __restrict__ prm, const double* __restrict__ dat, int robust,
                                    double* __restrict__ out) {
    if (threadIdx.x != 0) return;
    VisualEval e;
    // prm: pose_i 7 | pose_j 7 | ex 7 | inv_dep | td     dat: pts_i 2, pts_j 2, vel_i 2, vel_j 2, td_i, td_j, row_i, row_j
    eval_visual<true, true>(d, prm, prm + 7, prm + 14, prm[21], prm[22], dat[0], dat[1], dat[2], dat[3], dat[4], dat[5], dat[6], dat[7], dat[8],
                dat[9], dat[10], dat[11], true, robust != 0, e);
    out[0] = e.r[0];
    out[1] = e.r[1];
    for (int k = 0; k < 20; k++) {
        out[2 + k] = e.J[0][k];
        out[22 + k] = e.J[1][k];
    }
    out[42] = e.half_rho;
}

__global__ void __launch_bounds__(32) debug_imu_kernel(BaDims d, const PreInt* __restrict__ pre, const double* __restrict__ prm,
                                                       double* __restrict__ out) {
    __shared__ double Jraw[450], Jw[450], rr[15], rw[15];
    const int lane = threadIdx.x;
    for (int i = lane; i < 450; i += 32) Jraw[i] = 0.0;
    __syncwarp();
    // prm: pose_i 7 | sb_i 9 | pose_j 7 | sb_j 9
    if (lane == 0) eval_imu_raw(d, *pre, prm, prm + 7, prm + 16, prm + 23, rr, Jraw);
    __syncwarp();
    for (int idx = lane; idx < 450; idx += 32) {
        const int i = idx / 30, c = idx % 30;
        double s = 0;
        for (int k = 0; k < 15; k++) s += pre->sqrt_info[i * 15 + k] * Jraw[k * 30 + c];
        Jw[idx] = s;
    }
    if (lane < 15) {
        double s = 0;
        for (int k = 0; k < 15; k++) s += pre->sqrt_info[lane * 15 + k] * rr[k];
        rw[lane] = s;
    }
    __syncwarp();
    for (int i = lane; i < 15; i += 32) out[i] = rw[i];
    for (int i = lane; i < 450; i += 32) out[15 + i] = Jw[i];
}

}  // namespace vb

// ------------------------------------------------------------------------------------------------
// launch wrappers
namespace vb {

namespace {

// What the launches query of the current device: its opt-in shared-memory limit and the kernels' static shared sizes
// (handles may live on different GPUs of one process).
struct DeviceCfg {
    bool init = false;
    int smem_limit = 0, step_static = 0, marg_static = 0;
};
std::mutex g_cfg_mutex;
std::map<int, DeviceCfg> g_cfg;

DeviceCfg& device_cfg_locked() {  // caller holds g_cfg_mutex
    int dev = 0;
    cudaGetDevice(&dev);
    DeviceCfg& c = g_cfg[dev];
    if (!c.init) {
        cudaDeviceGetAttribute(&c.smem_limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cudaFuncAttributes fa{};
        cudaFuncGetAttributes(&fa, ba_step_kernel);
        c.step_static = (int)fa.sharedSizeBytes;
        cudaFuncGetAttributes(&fa, marg_solve_kernel);
        c.marg_static = (int)fa.sharedSizeBytes;
        c.init = true;
    }
    return c;
}

}  // namespace

int marg_w_in_global(int m_dense, int n) {
    std::lock_guard<std::mutex> lock(g_cfg_mutex);
    DeviceCfg& c = device_cfg_locked();
    return marg_solve_smem_bytes(m_dense, n, false) + (size_t)c.marg_static + 256 > (size_t)c.smem_limit ? 1 : 0;
}

void launch_preint_jobs(BaSeq* seqs, const BatchShape& sh, cudaStream_t s, int* launches, KernelProfile* prof) {
    KernelProfile none;
    if (!prof) prof = &none;
    if (!sh.any_jobs) return;
    prof->begin(s);
    preint_jobs_kernel<<<dim3(sh.W + 1, sh.S), 256, 0, s>>>(seqs);
    prof->end(6, s);
    if (launches) *launches += 1;
}

namespace {

void launch_eval(const BaSeq* seqs, const BatchShape& sh, int grid, int initial, cudaStream_t s) {
    const dim3 g(grid, sh.S);
    if (sh.est_ex && sh.est_td) ba_eval_kernel<true, true><<<g, 32 * LIN_WARPS, 0, s>>>(seqs, initial);
    else if (sh.est_ex) ba_eval_kernel<true, false><<<g, 32 * LIN_WARPS, 0, s>>>(seqs, initial);
    else if (sh.est_td) ba_eval_kernel<false, true><<<g, 32 * LIN_WARPS, 0, s>>>(seqs, initial);
    else ba_eval_kernel<false, false><<<g, 32 * LIN_WARPS, 0, s>>>(seqs, initial);
}

// Schur gather of every member: a CTA per pose-type block pair, incl. the relocalisation pose when a member of this frame has
// one (CTAs of pairs a member does not have return at once), then the CTAs of the generic entries
void launch_reduce(const BaSeq* seqs, const BatchShape& sh, cudaStream_t s) {
    const int NV = sh.W + 1 + (sh.est_ex ? 1 : 0) + (sh.est_td ? 1 : 0) + (sh.any_relo ? 1 : 0), n_pairs = NV * (NV + 1) / 2;
    const int generic = (sh.D * (sh.D + 1) / 2 + 4 * RED_THREADS - 1) / (4 * RED_THREADS);
    if (sh.any_relo) ba_reduce_kernel<true><<<dim3(n_pairs + generic, sh.S), RED_THREADS, 0, s>>>(seqs, n_pairs);
    else ba_reduce_kernel<false><<<dim3(n_pairs + generic, sh.S), RED_THREADS, 0, s>>>(seqs, n_pairs);
}

// Dynamic shared memory of marg_solve_kernel at the batch's maxima, with the kernel's opt-in on this device raised to it
size_t prepare_marg_solve(const BatchShape& sh) {
    const size_t smem = marg_solve_smem_bytes(sh.max_md, sh.max_n, sh.w_in_global != 0);
    raise_dynamic_smem((const void*)marg_solve_kernel, (int)smem);
    return smem;
}

}  // namespace

void launch_ba_solve(BaSeq* seqs, const BatchShape& sh, cudaStream_t s, int* launches, KernelProfile* prof) {
    KernelProfile none;
    if (!prof) prof = &none;
    if (!sh.any_active) return;
    BaDims dmax{};
    dmax.L = sh.max_L;
    dmax.W = sh.W;
    const int eval_grid = ba_eval_grid(dmax);
    const size_t panel_bytes = sizeof(double) * CHOL_NB * CHOL_PS;
    const size_t chol_bytes = sizeof(double) * (size_t)(sh.D + 1) * (sh.D + 2) / 2 + panel_bytes;
    int use_smem;
    {
        std::lock_guard<std::mutex> lock(g_cfg_mutex);
        DeviceCfg& c = device_cfg_locked();
        use_smem = chol_bytes + (size_t)c.step_static + 256 <= (size_t)c.smem_limit ? 1 : 0;
    }
    const size_t step_dyn = use_smem ? chol_bytes : panel_bytes;
    raise_dynamic_smem((const void*)ba_step_kernel, (int)step_dyn);
    int n = 0;
    prof->begin(s);
    launch_eval(seqs, sh, eval_grid, 1, s);
    prof->end(0, s);
    n += 1;
    for (int it = 0; it < sh.max_iterations; it++) {
        prof->begin(s);
        launch_reduce(seqs, sh, s);
        prof->end(1, s);
        prof->begin(s);
        ba_step_kernel<<<sh.S, 512, step_dyn, s>>>(seqs, use_smem);
        prof->end(2, s);
        prof->begin(s);
        launch_eval(seqs, sh, eval_grid, 0, s);
        prof->end(0, s);
        n += 3;
    }
    prof->begin(s);
    ba_finish_kernel<<<sh.S, 128, 0, s>>>(seqs);
    prof->end(7, s);
    n += 1;
    if (launches) *launches += n;
}

void launch_marginalize(BaSeq* seqs, const BatchShape& sh, cudaStream_t s, int* launches, KernelProfile* prof) {
    KernelProfile none;
    if (!prof) prof = &none;
    if (!sh.any_marg) return;
    const size_t smem = prepare_marg_solve(sh);
    const int zgrid = std::max(1, std::min(64, (int)(((size_t)sh.max_P * sh.max_P + 256 * 8 - 1) / (256 * 8))));
    const int egrid = (sh.max_n_lm + LIN_WARPS - 1) / LIN_WARPS + 2;
    const int dense_ctas = 16, lm_ctas = (sh.max_n_lm + 3) / 4;
    prof->begin(s);
    marg_zero_kernel<<<dim3(zgrid, sh.S), 256, 0, s>>>(seqs);
    if (sh.est_td) marg_eval_kernel<true><<<dim3(egrid, sh.S), 32 * LIN_WARPS, 0, s>>>(seqs);
    else marg_eval_kernel<false><<<dim3(egrid, sh.S), 32 * LIN_WARPS, 0, s>>>(seqs);
    marg_gather_kernel<<<dim3(dense_ctas + lm_ctas, sh.S), 128, 0, s>>>(seqs, dense_ctas);
    prof->end(4, s, 3);
    prof->begin(s);
    marg_solve_kernel<<<sh.S, MARG_THREADS, smem, s>>>(seqs, 1e-8);
    prof->end(5, s);
    if (launches) *launches += 4;
}

void launch_debug_visual(const BaDims& d, const double* d_params23, const double* d_data16, int robust, double* d_out, cudaStream_t s) {
    debug_visual_kernel<<<1, 32, 0, s>>>(d, d_params23, d_data16, robust, d_out);
}
void launch_debug_imu(const BaDims& d, const PreInt* d_pre, const double* d_params32, double* d_out, cudaStream_t s) {
    debug_imu_kernel<<<1, 32, 0, s>>>(d, d_pre, d_params32, d_out);
}

}  // namespace vb
