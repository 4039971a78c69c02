// 4-DoF pose-graph optimisation on the device: PoseGraph::optimize4DoF (pose_graph/src/pose_graph.cpp:403-579) solved by
// Ceres 1.14's Levenberg-Marquardt with the semantics csrc/initial.cpp's sfm_bundle restates (Jacobi scaling fixed at the
// first Jacobian, radius 1e4, the 1 - (2 rho - 1)^3 rule, diagonal clamp [1e-6, 1e32], function / parameter / gradient
// tolerances 1e-6 / 1e-8 / 1e-10).  float64 throughout, no atomics: every sum has a fixed order, so runs are
// bit-reproducible and a batch member computes exactly what a stand-alone handle computes.
//
// Parameters: per key frame of the range yaw (degrees, NormalizeAngle on update) and t; local key frames 0 .. nc - 1 are
// constant (the earliest loop anchor, or the key frames of a loaded map that share an edge with a free one; the host
// packs no edge between two constants, see pose_graph.cpp).  The damped normal equations are solved exactly with this
// structure:
//   chain   the free key frames in super-blocks of 4 by local index (16 unknowns each), from the super-block holding
//           local nc on: the super-blocks before it hold constants only.  Sequential edges reach back at most 4 key
//           frames, so their part of the system is block-tridiagonal.
//   border  the free loop anchors (old ends of loop edges), 4 columns each, D of them.  Their rows and columns are
//           identity rows in the chain; every loop edge has an end in the border or a constant end.
//   step 1  block Cholesky along the chain (pg_chain_kernel, ceil((D + 1) / 384) CTAs per member), carrying
//           W = L^-1 B and y = L^-1 (-g) as extra right-hand sides, one thread per border column.
//   step 2  S = C - W^T W and z = -g_b - W^T y, rows summed in ascending order; W is a staircase, each column starts at
//           its first coupled super-block.
//   step 3  the Cholesky of [S; z^T] (the z row gives the forward solve), the backward solve, then back-substitution
//           through the chain.
// Steps 2 and 3 take one of two routes per member, both in the same launch chain (each kernel returns early for the
// members of the other route):
//   D <= PG_MAX_D  pg_border_kernel (32 x 32 tiles into the packed system), pg_solve_kernel (cholesky_packed and
//                  chol_solve_packed in one CTA, in shared memory).
//   D >  PG_MAX_D  the multi-CTA path, in global memory on U (pg_layout.h): pg_tile_kernel<false> (S and z, one 64 x 64
//                  tile per CTA on FP64 tensor cores), per panel of 64 columns pg_panel_kernel (diagonal tile and the
//                  panel's row) and pg_tile_kernel<true> (the trailing update, the same tile product), then
//                  pg_solve_large_kernel (blocked backward solve and the chain's back-substitution).
#include "cuda_check.h"
#include "pg_kernels.h"
#include "pg_layout.h"

#include <algorithm>
#include <cfloat>
#include <climits>

#include "ba_device.cuh"
#include "chol_packed.cuh"

namespace vb {
namespace {

constexpr double PG_HUBER_A = 0.1;  // HuberLoss(0.1), pose_graph.cpp:440

// FourDOFError / FourDOFWeightError (pose_graph.h:159-248) between the older key frame i (yaw_i, pitch_i, roll_i) and the
// newer j; xi / xj = yaw (degrees), t.  meas = t_rel (3), yaw_rel.  J (may be NULL): 4 x 8, columns yaw_i, t_i, yaw_j,
// t_j, yaw in degrees.  With `robust` the HuberLoss(0.1) corrector (rho'' <= 0 branch: residual and Jacobian times
// sqrt(rho')) is applied.  Returns the cost 0.5 rho(|r|^2).
__device__ double four_dof_eval(const double* xi, const double* xj, double pitch_i, double roll_i, const double* meas, bool weighted,
                                bool robust, double* r, double* J) {
    const Mat3 R = ypr2R(Vec3(xi[0], pitch_i, roll_i));
    const double d0 = xj[1] - xi[1], d1 = xj[2] - xi[2], d2 = xj[3] - xi[3];
    for (int k = 0; k < 3; k++) r[k] = (R.m[k] * d0 + R.m[3 + k] * d1 + R.m[6 + k] * d2) - meas[k];
    r[3] = normalize_angle(xj[0] - xi[0] - meas[3]);
    if (weighted) r[3] = r[3] / 10.0;
    if (J) {
        const double c = M_PI / 180.0, w = weighted ? 0.1 : 1.0;
        // dR/dyaw = [[0,-1,0],[1,0,0],[0,0,0]] R: row 0 = -R row 1, row 1 = R row 0
        for (int k = 0; k < 3; k++) {
            J[8 * k] = c * (-R.m[3 + k] * d0 + R.m[k] * d1);
            for (int m = 0; m < 3; m++) {
                J[8 * k + 1 + m] = -R.m[3 * m + k];
                J[8 * k + 5 + m] = R.m[3 * m + k];
            }
            J[8 * k + 4] = 0.0;
        }
        for (int m = 0; m < 8; m++) J[24 + m] = 0.0;
        J[24] = -w;
        J[28] = w;
    }
    const double s = r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
    if (!robust) return 0.5 * s;
    const double b = PG_HUBER_A * PG_HUBER_A;
    double rho = s, rho1 = 1.0;
    if (s > b) {
        const double q = sqrt(s);
        rho = 2.0 * PG_HUBER_A * q - b;
        rho1 = fmax(DBL_MIN, PG_HUBER_A / q);
    }
    const double sc = sqrt(rho1);
    for (int k = 0; k < 4; k++) r[k] *= sc;
    if (J)
        for (int k = 0; k < 32; k++) J[k] *= sc;
    return 0.5 * rho;
}

struct PgView {
    int n, nb, nc, D, Dp, nsb;
    const double *pose, *loopm;
    const int *seq, *loop, *bslot, *lfirst, *lnext, *anchors;
    PgState* st;
    double *x, *xc, *dx, *scale, *ypr, *smeas, *blk, *g, *L, *F, *W, *Sp, *U, *Ud, *yb;
    int* start;
    int Np;
    double* out;
};

__device__ PgView pg_view(const PgLaunch& a, int slot) {
    const PgHdrLayout h = pg_hdr_layout(a.S);
    const int m = reinterpret_cast<const int*>(a.d_in + h.member)[slot];
    PgView v;
    v.n = reinterpret_cast<const int*>(a.d_in + h.n)[slot];
    v.nb = reinterpret_cast<const int*>(a.d_in + h.nb)[slot];
    v.nc = reinterpret_cast<const int*>(a.d_in + h.nc)[slot];
    v.D = 4 * v.nb;
    v.Dp = v.D + 1;
    v.nsb = pg_num_sb(v.n);
    const char* in = a.d_in + reinterpret_cast<const long long*>(a.d_in + h.in_off)[slot];
    const PgInLayout il = pg_in_layout(v.n, v.nb);
    v.pose = reinterpret_cast<const double*>(in + il.pose);
    v.loopm = reinterpret_cast<const double*>(in + il.loop);
    v.seq = reinterpret_cast<const int*>(in + il.seq);
    v.loop = reinterpret_cast<const int*>(in + il.loop_idx);
    v.bslot = reinterpret_cast<const int*>(in + il.bslot);
    v.lfirst = reinterpret_cast<const int*>(in + il.lfirst);
    v.lnext = reinterpret_cast<const int*>(in + il.lnext);
    v.anchors = reinterpret_cast<const int*>(in + il.anchors);
    double* w = a.d_work + (size_t)m * a.work_stride;
    const PgWorkLayout wl = pg_work_layout(a.cap_n, a.cap_anchors);
    v.st = reinterpret_cast<PgState*>(w + wl.state);
    v.x = w + wl.x; v.xc = w + wl.xc; v.dx = w + wl.dx; v.scale = w + wl.scale; v.ypr = w + wl.ypr; v.smeas = w + wl.smeas;
    v.blk = w + wl.blk; v.g = w + wl.g; v.L = w + wl.L; v.F = w + wl.F; v.W = w + wl.W; v.Sp = w + wl.Sp;
    v.U = w + wl.U; v.Ud = w + wl.Ud; v.yb = w + wl.yb;
    v.Np = pg_tile_np(v.D);
    v.start = reinterpret_cast<int*>(w + wl.start);
    v.out = a.d_out + reinterpret_cast<const long long*>(a.d_in + h.out_off)[slot];
    return v;
}

// kind of a local key frame: 0 chain (free, not an anchor), 1 border (free anchor), 2 constant (local < nc), 3 padding
__device__ __forceinline__ int kf_kind(const PgView& v, int k) {
    if (k >= v.n) return 3;
    if (k < v.nc) return 2;
    return v.bslot[k] >= 0 ? 1 : 0;
}

// The edges a key frame owns as their newer end: e = 0..3 sequential to a - e - 1, e = 4 its loop edge.
__device__ __forceinline__ int edge_older(const PgView& v, int a, int e) {
    if (e < 4) {
        const int b = a - e - 1;
        return (b >= 0 && v.seq[b] == v.seq[a]) ? b : -1;
    }
    return v.loop[a];
}
__device__ __forceinline__ double edge_eval(const PgView& v, const double* x, int a, int e, int b, double* r, double* J) {
    const double* meas = e < 4 ? v.smeas + 16 * a + 4 * e : v.loopm + 4 * a;
    return four_dof_eval(x + 4 * b, x + 4 * a, v.ypr[3 * b + 1], v.ypr[3 * b + 2], meas, e == 4, e == 4, r, J);
}

__device__ __forceinline__ double block_sum_d(double val, double* red) {
    val = warp_sum_d(val);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = val;
    __syncthreads();
    double s = 0;
    for (unsigned w = 0; w < blockDim.x / 32; w++) s += red[w];
    __syncthreads();
    return s;
}

// cost of every edge at point x, summed per thread in key-frame order and then across the CTA in a fixed order
__device__ double total_cost(const PgView& v, const double* x, double* red) {
    double part = 0;
    for (int a = threadIdx.x; a < v.n; a += blockDim.x)
        for (int e = 0; e < 5; e++) {
            const int b = edge_older(v, a, e);
            if (b < 0) continue;
            double r[4];
            part += edge_eval(v, x, a, e, b, r, nullptr);
        }
    return block_sum_d(part, red);
}

// ---- setup: initial point (yaw from R2ypr of the VIO rotation), constant pitch / roll, sequential measurements
//      (pose_graph.cpp:447-495), state, initial cost
__global__ void __launch_bounds__(256) pg_setup_kernel(PgLaunch a) {
    __shared__ double red[8];
    const PgView v = pg_view(a, blockIdx.x);
    for (int k = threadIdx.x; k < v.n; k += blockDim.x) {
        const double* p = v.pose + 7 * k;
        const Vec3 ypr = R2ypr(qR(Quat{p[3], p[4], p[5], p[6]}));
        v.ypr[3 * k] = ypr.x; v.ypr[3 * k + 1] = ypr.y; v.ypr[3 * k + 2] = ypr.z;
        v.x[4 * k] = ypr.x; v.x[4 * k + 1] = p[0]; v.x[4 * k + 2] = p[1]; v.x[4 * k + 3] = p[2];
    }
    __syncthreads();
    for (int k = threadIdx.x; k < v.n; k += blockDim.x)
        for (int e = 0; e < 4; e++) {
            const int b = edge_older(v, k, e);
            double* m = v.smeas + 16 * k + 4 * e;
            if (b < 0) { m[0] = m[1] = m[2] = m[3] = 0.0; continue; }
            const double* pb = v.pose + 7 * b;
            const Mat3 Rb = qR(Quat{pb[3], pb[4], pb[5], pb[6]});
            const double d0 = v.x[4 * k + 1] - v.x[4 * b + 1], d1 = v.x[4 * k + 2] - v.x[4 * b + 2], d2 = v.x[4 * k + 3] - v.x[4 * b + 3];
            for (int c = 0; c < 3; c++) m[c] = Rb.m[c] * d0 + Rb.m[3 + c] * d1 + Rb.m[6 + c] * d2;
            m[3] = v.x[4 * k] - v.x[4 * b];
        }
    __syncthreads();
    const double cost = total_cost(v, v.x, red);
    if (threadIdx.x == 0) {
        PgState s{};
        s.radius = 1e4; s.decrease = 2.0; s.cost = cost; s.cost0 = cost;
        s.need_lin = 1; s.first = 1;
        s.done = (v.n < 2 || !isfinite(cost)) ? 1 : 0;
        *v.st = s;
    }
}

// ---- linearise (only after an accepted step): per key frame its diagonal block, the blocks to the key frames 1..4 back
//      (a loop edge onto one of them is merged in), its loop block, the gradient; Jacobi scaling on the first call;
//      gradient tolerance.  Each block gathers its edges in a fixed order: own sequential edges, own loop edge,
//      sequential edges of the 4 newer key frames, incoming loop edges by ascending source.
__global__ void __launch_bounds__(256) pg_linearize_kernel(PgLaunch a) {
    __shared__ double red[8];
    const PgView v = pg_view(a, blockIdx.x);
    if (v.st->done || !v.st->need_lin) return;
    double* ej = v.W;  // edge scratch (W is free until the chain kernel): per key frame 5 x (r 4 | J 32)
    for (int k = threadIdx.x; k < v.n; k += blockDim.x)
        for (int e = 0; e < 5; e++) {
            const int b = edge_older(v, k, e);
            if (b >= 0) edge_eval(v, v.x, k, e, b, ej + 180 * k + 36 * e, ej + 180 * k + 36 * e + 4);
        }
    __syncthreads();
    double gmax = 0;
    for (int k = threadIdx.x; k < v.n; k += blockDim.x) {
        double H[16] = {}, g[4] = {}, B[4][16] = {}, Lb[16] = {};
        auto add_newer = [&](const double* rj, double* Hb, const double* r) {  // k is the newer end (columns 4..7)
            const double* J = rj;
            for (int p = 0; p < 4; p++) {
                for (int q = 0; q < 4; q++) {
                    double s = 0;
                    for (int t = 0; t < 4; t++) s += J[8 * t + 4 + p] * J[8 * t + 4 + q];
                    H[4 * p + q] += s;
                }
                double s = 0;
                for (int t = 0; t < 4; t++) s += J[8 * t + 4 + p] * r[t];
                g[p] += s;
                for (int q = 0; q < 4; q++) {
                    double o = 0;
                    for (int t = 0; t < 4; t++) o += J[8 * t + 4 + p] * J[8 * t + q];
                    Hb[4 * p + q] += o;
                }
            }
        };
        auto add_older = [&](const double* r, const double* J) {  // k is the older end (columns 0..3)
            for (int p = 0; p < 4; p++) {
                for (int q = 0; q < 4; q++) {
                    double s = 0;
                    for (int t = 0; t < 4; t++) s += J[8 * t + p] * J[8 * t + q];
                    H[4 * p + q] += s;
                }
                double s = 0;
                for (int t = 0; t < 4; t++) s += J[8 * t + p] * r[t];
                g[p] += s;
            }
        };
        for (int e = 0; e < 4; e++)
            if (edge_older(v, k, e) >= 0) add_newer(ej + 180 * k + 36 * e + 4, B[e], ej + 180 * k + 36 * e);
        const int lt = v.loop[k];
        if (lt >= 0) add_newer(ej + 180 * k + 36 * 4 + 4, (k - lt <= 4) ? B[k - lt - 1] : Lb, ej + 180 * k + 36 * 4);
        for (int e = 0; e < 4; e++) {
            const int j = k + e + 1;
            if (j < v.n && edge_older(v, j, e) == k) add_older(ej + 180 * j + 36 * e, ej + 180 * j + 36 * e + 4);
        }
        for (int j = v.lfirst[k]; j >= 0; j = v.lnext[j]) add_older(ej + 180 * j + 36 * 4, ej + 180 * j + 36 * 4 + 4);
        double* o = v.blk + (size_t)PG_BLK_KF * k;
        for (int t = 0; t < 16; t++) {
            o[PG_BLK_DIAG + t] = H[t];
            o[PG_BLK_LOOP + t] = Lb[t];
            for (int e = 0; e < 4; e++) o[PG_BLK_BACK + 16 * e + t] = B[e][t];
        }
        for (int p = 0; p < 4; p++) {
            v.g[4 * k + p] = g[p];
            if (k >= v.nc) gmax = fmax(gmax, fabs(g[p]));
            if (v.st->first) v.scale[4 * k + p] = 1.0 / (1.0 + sqrt(H[5 * p]));
        }
    }
    // max over the CTA (order-free)
    gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 16));
    gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 8));
    gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 4));
    gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 2));
    gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 1));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = gmax;
    __syncthreads();
    for (int k = threadIdx.x; k < v.n; k += blockDim.x) {  // scaled system: H_ij s_i s_j, g_i s_i
        const double* sk = v.scale + 4 * k;
        double* o = v.blk + (size_t)PG_BLK_KF * k;
        for (int p = 0; p < 4; p++) {
            v.g[4 * k + p] *= sk[p];
            for (int q = 0; q < 4; q++) o[PG_BLK_DIAG + 4 * p + q] *= sk[p] * sk[q];
            for (int e = 0; e < 4; e++)
                if (k - e - 1 >= 0)
                    for (int q = 0; q < 4; q++) o[PG_BLK_BACK + 16 * e + 4 * p + q] *= sk[p] * v.scale[4 * (k - e - 1) + q];
            if (v.loop[k] >= 0)
                for (int q = 0; q < 4; q++) o[PG_BLK_LOOP + 4 * p + q] *= sk[p] * v.scale[4 * v.loop[k] + q];
        }
    }
    if (threadIdx.x == 0) {
        double m = 0;
        for (unsigned w = 0; w < blockDim.x / 32; w++) m = fmax(m, red[w]);
        PgState* s = v.st;
        s->gmax = m;
        s->first = 0;
        s->need_lin = 0;
        if (m <= 1e-10) s->done = s->converged = 1;
    }
}

// H(ka, kb) entry (p, q) of the scaled system between two free key frames (0 when no edge joins them)
__device__ __forceinline__ double h_entry(const PgView& v, int ka, int kb, int p, int q) {
    if (ka == kb) return v.blk[(size_t)PG_BLK_KF * ka + PG_BLK_DIAG + 4 * p + q];
    if (ka < kb) { const int t = ka; ka = kb; kb = t; const int u = p; p = q; q = u; }
    if (ka - kb <= 4) return v.blk[(size_t)PG_BLK_KF * ka + PG_BLK_BACK + 16 * (ka - kb - 1) + 4 * p + q];
    if (v.loop[ka] == kb) return v.blk[(size_t)PG_BLK_KF * ka + PG_BLK_LOOP + 4 * p + q];
    return 0.0;
}
__device__ __forceinline__ double damped(double h, double radius) { return h + fmin(fmax(h, 1e-6), 1e32) / radius; }

// ---- step 1: block Cholesky along the chain; thread c < D + 1 carries border column c (c = D: the right-hand side).
//      The columns spread over ceil((D + 1) / 384) CTAs (grid.x; grid.y is the member slot).  Every CTA repeats the
//      super-block factorisation, which is deterministic, so all compute the same bits; CTA 0 alone stores L and F.
//      The chain starts at super-block s0 = nc / 4: the earlier ones are identity blocks that couple to nothing (their
//      F blocks into s0 are zero), so neither L, F nor W is formed for them.
__global__ void __launch_bounds__(384) pg_chain_kernel(PgLaunch a) {
    __shared__ double Lp[16][17], Lc[16][17], Fs[16][17], M[16][17];
    __shared__ int fail;
    const PgView v = pg_view(a, blockIdx.y);
    if (v.st->done || (int)(blockIdx.x * blockDim.x) >= v.Dp) return;
    const bool writer = blockIdx.x == 0;
    const double radius = v.st->radius;
    const int tid = threadIdx.x, c = blockIdx.x * blockDim.x + tid;
    const bool col = c < v.Dp;
    int bk = -1, bq = 0;
    if (col && c < v.D) { bk = v.anchors[c >> 2]; bq = c & 3; }
    double w[16];
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = 0.0;
    bool started = false;
    int start = v.nsb;
    const int s0 = v.nc / PG_SB;
    if (tid == 0) fail = 0;
    for (int s = s0; s < v.nsb; s++) {
        for (int e = tid; e < 256; e += blockDim.x) {
            const int r = e >> 4, cc = e & 15, ka = 4 * s + (r >> 2), kb = 4 * s + (cc >> 2), kc = 4 * (s - 1) + (cc >> 2);
            double m = (r == cc) ? 1.0 : 0.0;
            if (kf_kind(v, ka) == 0 && kf_kind(v, kb) == 0) {
                m = h_entry(v, ka, kb, r & 3, cc & 3);
                if (r == cc) m = damped(m, radius);
            }
            M[r][cc] = m;
            Fs[r][cc] = (s > 0 && kf_kind(v, ka) == 0 && kf_kind(v, kc) == 0 && ka - kc <= 4) ? h_entry(v, ka, kc, r & 3, cc & 3) : 0.0;
        }
        __syncthreads();
        if (s > s0) {
            if (tid < 16) {  // F = E L_{s-1}^-T, one row per thread
                const int r = tid;
                for (int q = 0; q < 16; q++) {
                    double val = Fs[r][q];
                    for (int t = 0; t < q; t++) val -= Fs[r][t] * Lp[q][t];
                    Fs[r][q] = val / Lp[q][q];
                }
            }
            __syncthreads();
            for (int e = tid; e < 256; e += blockDim.x) {
                const int r = e >> 4, q = e & 15;
                if (writer) v.F[256 * s + e] = Fs[r][q];
                if (q <= r) {
                    double acc = 0;
                    for (int t = 0; t < 16; t++) acc += Fs[r][t] * Fs[q][t];
                    M[r][q] -= acc;
                }
            }
            __syncthreads();
        }
        if (tid < 32) {  // 16 x 16 Cholesky, one row per lane
            const int r = tid & 15;
            double row[16];
#pragma unroll
            for (int q = 0; q < 16; q++) row[q] = M[r][q];
            bool ok = true;
#pragma unroll
            for (int q = 0; q < 16; q++) {
                const double piv = __shfl_sync(0xffffffffu, row[q], q);
                if (!(piv > 0.0) || !isfinite(piv)) ok = false;
                const double d = sqrt(piv);
                if (r > q) row[q] /= d;
                if (r == q) row[q] = d;
                const double lrq = row[q];
#pragma unroll
                for (int k = q + 1; k < 16; k++) {
                    const double lkq = __shfl_sync(0xffffffffu, lrq, k);
                    if (r >= k) row[k] -= lrq * lkq;
                }
            }
            if (tid < 16) {
#pragma unroll
                for (int q = 0; q < 16; q++) {
                    const double val = q <= r ? row[q] : 0.0;
                    Lc[r][q] = val;
                    if (writer) v.L[256 * s + 16 * r + q] = val;
                }
                if (!ok) fail = 1;
            }
        }
        __syncthreads();
        if (fail) break;
        if (col) {
            double b[16];
            bool nz = false;
#pragma unroll
            for (int k = 0; k < 16; k++) {
                const int kf = 4 * s + (k >> 2);
                double val = 0.0;
                if (kf_kind(v, kf) == 0) val = (c == v.D) ? -v.g[4 * kf + (k & 3)] : h_entry(v, kf, bk, k & 3, bq);
                b[k] = val;
                nz |= val != 0.0;
            }
            if (!started && nz) { started = true; start = s; }
            if (started) {
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    double val = b[k];
                    if (s > s0)
#pragma unroll
                        for (int t = 0; t < 16; t++) val -= Fs[k][t] * w[t];
                    b[k] = val;
                }
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    double val = b[k];
#pragma unroll
                    for (int t = 0; t < k; t++) val -= Lc[k][t] * w[t];
                    w[k] = val / Lc[k][k];
                }
#pragma unroll
                for (int k = 0; k < 16; k++) v.W[(size_t)(16 * s + k) * v.Dp + c] = w[k];
            }
        }
        __syncthreads();
        for (int e = tid; e < 256; e += blockDim.x) Lp[e >> 4][e & 15] = Lc[e >> 4][e & 15];
        __syncthreads();
    }
    if (col) v.start[c] = started ? start : v.nsb;
    if (writer && tid == 0 && fail) v.st->lin_fail = 1;
}

// ---- step 2: the border system [S; z^T] packed (row D = z), one 32 x 32 tile per CTA, W rows in ascending order
__global__ void __launch_bounds__(256) pg_border_kernel(PgLaunch a) {
    __shared__ double Wa[64][33], Wb[64][33];
    const PgView v = pg_view(a, blockIdx.y);
    if (v.st->done || v.st->lin_fail || v.D == 0 || v.D > PG_MAX_D) return;
    const int T = (v.Dp + 31) / 32, t = blockIdx.x;
    if (t >= T * (T + 1) / 2) return;
    int ti = 0;
    while ((ti + 1) * (ti + 2) / 2 <= t) ti++;
    const int tj = t - ti * (ti + 1) / 2, r0 = 32 * ti, c0 = 32 * tj;
    const double radius = v.st->radius;
    const int rows = 16 * v.nsb, Dp = v.Dp, D = v.D;
    int est[4];
    double acc[4] = {0, 0, 0, 0};
    int first = v.nsb;
    for (int k = 0; k < 32; k++) {
        if (r0 + k < Dp) first = min(first, v.start[r0 + k]);
    }
    int firstc = v.nsb;
    for (int k = 0; k < 32; k++)
        if (c0 + k < Dp) firstc = min(firstc, v.start[c0 + k]);
    first = 16 * max(first, firstc);
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int e = threadIdx.x + 256 * q, r = r0 + (e >> 5), cc = c0 + (e & 31);
        est[q] = (r < Dp && cc < Dp) ? 16 * max(v.start[r], v.start[cc]) : rows;
    }
    for (int ch = first; ch < rows; ch += 64) {
        for (int e = threadIdx.x; e < 64 * 32; e += blockDim.x) {
            const int rr = e >> 5, k = e & 31, row = ch + rr;
            Wa[rr][k] = (row < rows && r0 + k < Dp) ? v.W[(size_t)row * Dp + r0 + k] : 0.0;
            Wb[rr][k] = (row < rows && c0 + k < Dp) ? v.W[(size_t)row * Dp + c0 + k] : 0.0;
        }
        __syncthreads();
        const int lim = min(64, rows - ch);
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int e = threadIdx.x + 256 * q, lr = e >> 5, lc = e & 31;
            for (int rr = max(0, est[q] - ch); rr < lim; rr++) acc[q] += Wa[rr][lr] * Wb[rr][lc];
        }
        __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int e = threadIdx.x + 256 * q, r = r0 + (e >> 5), cc = c0 + (e & 31);
        if (r >= Dp || cc >= D || cc > r) continue;
        const int kq = v.anchors[cc >> 2];
        double h;
        if (r == D) {
            h = -v.g[4 * kq + (cc & 3)];
        } else {
            h = h_entry(v, v.anchors[r >> 2], kq, r & 3, cc & 3);
            if (r == cc) h = damped(h, radius);
        }
        v.Sp[(size_t)r * (r + 1) / 2 + cc] = h - acc[q];
    }
}

// Back-substitution through the chain for a member whose border step yb (scaled) is known: the step (unscaled) into dx.
// The 16 x 16 blocks and vectors are the caller's shared memory.
__device__ __forceinline__ void chain_back_substitute(const PgView& v, const double* yb, double (*Ls)[17], double (*Fn)[17], double* xs,
                                                      double* xn, double* rhs) {
    const int tid = threadIdx.x, D = v.D, Dp = v.Dp;
    if (tid < 16) xn[tid] = 0.0;
    const int wid = tid >> 5, lane = tid & 31;
    for (int s = v.nsb - 1; s >= v.nc / PG_SB; s--) {
        for (int e = tid; e < 256; e += blockDim.x) {
            Ls[e >> 4][e & 15] = v.L[256 * s + e];
            Fn[e >> 4][e & 15] = (s + 1 < v.nsb) ? v.F[256 * (s + 1) + e] : 0.0;
        }
        __syncthreads();
        if (wid < 16) {  // rhs_k = y_k - (W delta_b)_k - (F_{s+1}^T x_{s+1})_k, one warp per row
            const int k = wid;
            const size_t row = (size_t)(16 * s + k) * Dp;
            double part = 0;
            for (int c = lane; c < D; c += 32)
                if (v.start[c] <= s) part += v.W[row + c] * yb[c];
            part = warp_sum_d(part);
            if (lane == 0) {
                double val = v.start[D] <= s ? v.W[row + D] : 0.0;
                val -= part;
                for (int m = 0; m < 16; m++) val -= Fn[m][k] * xn[m];
                rhs[k] = val;
            }
        }
        __syncthreads();
        if (tid < 32) {  // L^T x = rhs, one row per lane, columns from the last
            const int k = tid & 15;
            double rk = rhs[k], xk = 0.0;
            for (int q = 15; q >= 0; q--) {
                const double xq = __shfl_sync(0xffffffffu, rk / Ls[q][q], q);
                if (k == q) xk = xq;
                if (k < q) rk -= Ls[q][k] * xq;
            }
            if (tid < 16) xs[k] = xk;
        }
        __syncthreads();
        if (tid < 16) {
            const int kf = 4 * s + (tid >> 2), p = tid & 3;
            const int kind = kf_kind(v, kf);
            if (kind != 3) {
                double d = 0.0;
                if (kind == 0) d = xs[tid];
                else if (kind == 1) d = yb[4 * v.bslot[kf] + p];
                v.dx[4 * kf + p] = d * v.scale[4 * kf + p];
            }
            xn[tid] = xs[tid];
        }
        __syncthreads();
    }
}

// ---- step 3: factor the border system, solve it, back-substitute through the chain; the step (unscaled) into dx
__global__ void __launch_bounds__(512) pg_solve_kernel(PgLaunch a) {
    extern __shared__ __align__(16) double pg_panel[];  // CHOL_NB * CHOL_PS
    __shared__ double rdiag[PG_MAX_D], yb[PG_MAX_D], linv[(PG_MAX_D / CHOL_NB) * 64];
    __shared__ double Ls[16][17], Fn[16][17], xs[16], xn[16], rhs[16];
    __shared__ int flag;
    const PgView v = pg_view(a, blockIdx.x);
    if (v.st->done || v.st->lin_fail || v.D > PG_MAX_D) return;
    const int tid = threadIdx.x, D = v.D;
    if (D > 0) {
        const bool ok = cholesky_packed(v.Sp, pg_panel, D, rdiag, linv, &flag, D + 1);
        if (!ok) {
            if (tid == 0) v.st->lin_fail = 1;
            return;
        }
        for (int c = tid; c < D; c += blockDim.x) yb[c] = v.Sp[(size_t)D * (D + 1) / 2 + c];
        __syncthreads();
        chol_solve_packed(v.Sp, linv, D, yb, false);
        __syncthreads();
    }
    chain_back_substitute(v, yb, Ls, Fn, xs, xn, rhs);
}

// ---- the multi-CTA path (D > PG_MAX_D).  U holds the upper triangle of [S z] (z in column D; rows and columns past D
//      are padding, 1 on the diagonal and 0 elsewhere), PG_TILE x PG_TILE tiles, Np = v.Np columns.  Right-looking
//      blocked Cholesky U = R^T R, panel p = rows / columns [64 p, 64 p + 64): the diagonal tile's factor goes to Ud, the
//      panel's row right of it becomes R's (including R^-T z = the forward solve, in column D), and the trailing tiles
//      are updated by the same tile product that forms S.

// FP64 tensor-core MMA m8n8k4, d = a b + d.  Fragments (PTX ISA, mma.m8n8k4 with .f64): a = A[lane / 4][lane % 4],
// b = B[lane % 4][lane / 4], d[e] = D[lane / 4][2 (lane % 4) + e].
__device__ __forceinline__ void mma_f64_m8n8k4(double* d, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
}

constexpr int PG_TK = 32;           // rows of X per shared-memory stage
constexpr int PG_TS = PG_TILE + 4;  // padded stage row: the fragment loads hit 16 distinct 8-byte banks per half-warp

// acc = X[k0:k1, i0:i0+64]^T X[k0:k1, j0:j0+64] over the rows in ascending order (stages of PG_TK rows, 4 rows per MMA).
// X is row-major with leading dimension ld; columns >= ncols read as 0, and with kstart != NULL so does every row below
// 16 kstart[column] (W's staircase: those rows are not written by the chain kernel).  256 threads: warp w owns rows
// 32 (w / 4) + 8 mt and columns 16 (w % 4) + 8 nt of the tile; acc[mt][nt][e] is its MMA fragment.
__device__ __forceinline__ void tile_product(const double* X, size_t ld, int k0, int k1, int i0, int j0, int ncols, const int* kstart,
                                             double (*Xa)[PG_TS], double (*Xb)[PG_TS], double (&acc)[4][2][2]) {
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, lc = tid & (PG_TILE - 1);
    const int ca = i0 + lc, cb = j0 + lc;
    const int ka = ca < ncols ? (kstart ? 16 * kstart[ca] : 0) : INT_MAX;
    const int kb = cb < ncols ? (kstart ? 16 * kstart[cb] : 0) : INT_MAX;
#pragma unroll
    for (int mt = 0; mt < 4; mt++)
#pragma unroll
        for (int nt = 0; nt < 2; nt++) acc[mt][nt][0] = acc[mt][nt][1] = 0.0;
    const int m0 = 32 * (w >> 2) + (lane >> 2), n0 = 16 * (w & 3) + (lane >> 2), kl = lane & 3;
    for (int ch = k0; ch < k1; ch += PG_TK) {
#pragma unroll
        for (int q = 0; q < PG_TK * PG_TILE / 256; q++) {
            const int rr = (tid >> 6) + 4 * q, k = ch + rr;
            Xa[rr][lc] = (k < k1 && k >= ka) ? X[(size_t)k * ld + ca] : 0.0;
            Xb[rr][lc] = (k < k1 && k >= kb) ? X[(size_t)k * ld + cb] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < PG_TK; kk += 4) {
            double fa[4], fb[2];
#pragma unroll
            for (int mt = 0; mt < 4; mt++) fa[mt] = Xa[kk + kl][m0 + 8 * mt];
#pragma unroll
            for (int nt = 0; nt < 2; nt++) fb[nt] = Xb[kk + kl][n0 + 8 * nt];
#pragma unroll
            for (int mt = 0; mt < 4; mt++)
#pragma unroll
                for (int nt = 0; nt < 2; nt++) mma_f64_m8n8k4(acc[mt][nt], fa[mt], fb[nt]);
        }
        __syncthreads();
    }
}

// ---- tiles of U's upper triangle, one per CTA (grid.x; grid.y is the member slot).
//      kTrailing = false (p unused): U = [C z] - W^T [W y], rows of W from the tile's first coupled super-block on.
//      kTrailing = true: after panel p, U_IJ -= R_pI^T R_pJ for the tiles p < I <= J.
template <bool kTrailing>
__global__ void __launch_bounds__(256) pg_tile_kernel(PgLaunch a, int p) {
    __shared__ __align__(16) double Xa[PG_TK][PG_TS], Xb[PG_TK][PG_TS];
    const PgView v = pg_view(a, blockIdx.y);
    if (v.st->done || v.st->lin_fail || v.D <= PG_MAX_D) return;
    const int base = kTrailing ? p + 1 : 0, R = v.Np / PG_TILE - base, t = blockIdx.x;
    if (t >= R * (R + 1) / 2) return;
    int ti = 0;
    while ((ti + 1) * (ti + 2) / 2 <= t) ti++;
    const int i0 = PG_TILE * (base + t - ti * (ti + 1) / 2), j0 = PG_TILE * (base + ti);  // i0 <= j0
    const size_t Np = v.Np;
    const int D = v.D, Dp = v.Dp, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double acc[4][2][2];
    if (kTrailing) {
        tile_product(v.U + (size_t)PG_TILE * p * Np, Np, 0, PG_TILE, i0, j0, (int)Np, nullptr, Xa, Xb, acc);
    } else {
        int fa = v.nsb, fb = v.nsb;
        for (int k = 0; k < PG_TILE; k++) {
            if (i0 + k < Dp) fa = min(fa, v.start[i0 + k]);
            if (j0 + k < Dp) fb = min(fb, v.start[j0 + k]);
        }
        tile_product(v.W, Dp, 16 * max(fa, fb), 16 * v.nsb, i0, j0, Dp, v.start, Xa, Xb, acc);
    }
    const double radius = v.st->radius;
#pragma unroll
    for (int mt = 0; mt < 4; mt++)
#pragma unroll
        for (int nt = 0; nt < 2; nt++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int i = i0 + 32 * (w >> 2) + 8 * mt + (lane >> 2), j = j0 + 16 * (w & 3) + 8 * nt + 2 * (lane & 3) + e;
                if (i > j) continue;
                double* u = v.U + (size_t)i * Np + j;
                if (kTrailing) {
                    *u -= acc[mt][nt][e];
                } else if (i < D && j <= D) {
                    const int ki = v.anchors[i >> 2];
                    double h;
                    if (j == D) {
                        h = -v.g[4 * ki + (i & 3)];
                    } else {
                        h = h_entry(v, ki, v.anchors[j >> 2], i & 3, j & 3);
                        if (i == j) h = damped(h, radius);
                    }
                    *u = h - acc[mt][nt][e];
                } else {
                    *u = i == j ? 1.0 : 0.0;
                }
            }
}

// ---- panel p: CTA c (grid.x) factors the diagonal tile U_pp = R_pp^T R_pp in shared memory (every CTA, the same bits)
//      and, for c > 0, solves R_pp^T R_p,p+c = U_p,p+c in place, right-looking by rows.  CTA 0 stores R_pp in Ud (the
//      other CTAs still read U_pp) and flags a pivot below D that is not positive and finite, as cholesky_packed does;
//      pivots at and past D (the z column and the padding) are taken as 1.
constexpr size_t PG_PANEL_SMEM = 2 * sizeof(double) * PG_TILE * (PG_TILE + 1);  // Rd | B, above the 48 KB default

__global__ void __launch_bounds__(256) pg_panel_kernel(PgLaunch a, int p) {
    extern __shared__ __align__(16) double pg_panel_tiles[];
    double(*Rd)[PG_TILE + 1] = reinterpret_cast<double(*)[PG_TILE + 1]>(pg_panel_tiles);
    double(*B)[PG_TILE + 1] = Rd + PG_TILE;
    __shared__ int bad;
    const PgView v = pg_view(a, blockIdx.y);
    if (v.st->done || v.D <= PG_MAX_D) return;
    const int c = blockIdx.x, tid = threadIdx.x;
    if (p + c >= v.Np / PG_TILE) return;
    const size_t Np = v.Np;
    const double* Upp = v.U + (size_t)PG_TILE * p * Np + PG_TILE * p;
    double* Ub = v.U + (size_t)PG_TILE * p * Np + PG_TILE * (p + c);
    for (int e = tid; e < PG_TILE * PG_TILE; e += blockDim.x) {
        const int r = e / PG_TILE, q = e % PG_TILE;
        Rd[r][q] = q >= r ? Upp[r * Np + q] : 0.0;
        if (c) B[r][q] = Ub[r * Np + q];
    }
    if (tid == 0) bad = 0;
    __syncthreads();
    for (int k = 0; k < PG_TILE; k++) {
        const double pk = Rd[k][k];
        const bool real = PG_TILE * p + k < v.D;
        const double d = real ? sqrt(pk) : 1.0;
        if (tid == 0 && real && (!(pk > 0.0) || !isfinite(pk))) bad = 1;
        __syncthreads();
        for (int j = k + tid; j < PG_TILE; j += blockDim.x) Rd[k][j] = j == k ? d : Rd[k][j] / d;
        if (c)
            for (int j = tid; j < PG_TILE; j += blockDim.x) B[k][j] /= d;
        __syncthreads();
        for (int e = tid; e < PG_TILE * PG_TILE; e += blockDim.x) {
            const int i = e / PG_TILE, j = e % PG_TILE;
            if (i <= k) continue;
            if (j >= i) Rd[i][j] -= Rd[k][i] * Rd[k][j];
            if (c) B[i][j] -= Rd[k][i] * B[k][j];
        }
        __syncthreads();
    }
    if (c) {
        for (int e = tid; e < PG_TILE * PG_TILE; e += blockDim.x) Ub[(e / PG_TILE) * Np + e % PG_TILE] = B[e / PG_TILE][e % PG_TILE];
    } else {
        double* ud = v.Ud + (size_t)PG_TILE * PG_TILE * p;
        for (int e = tid; e < PG_TILE * PG_TILE; e += blockDim.x) ud[e] = Rd[e / PG_TILE][e % PG_TILE];
        if (tid == 0 && bad) v.st->lin_fail = 1;
    }
}

// ---- step 3 of the multi-CTA path: R x = R^-T z by panels from the last (the rows' sums over the later panels one warp
//      per row, the diagonal tile by one warp from its last row), x = the border step into yb; then the chain.
__global__ void __launch_bounds__(512) pg_solve_large_kernel(PgLaunch a) {
    __shared__ double Rs[PG_TILE][PG_TILE + 1], rs[PG_TILE];
    __shared__ double Ls[16][17], Fn[16][17], xs[16], xn[16], rhs[16];
    const PgView v = pg_view(a, blockIdx.x);
    if (v.st->done || v.st->lin_fail || v.D <= PG_MAX_D) return;
    const int tid = threadIdx.x, D = v.D, wid = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
    const size_t Np = v.Np;
    for (int p = (D - 1) / PG_TILE; p >= 0; p--) {
        const int r0 = PG_TILE * p, nr = min(PG_TILE, D - r0);
        const double* ud = v.Ud + (size_t)PG_TILE * PG_TILE * p;
        for (int e = tid; e < PG_TILE * PG_TILE; e += blockDim.x) Rs[e / PG_TILE][e % PG_TILE] = ud[e];
        __syncthreads();
        for (int i = wid; i < nr; i += nw) {
            const double* Ri = v.U + (size_t)(r0 + i) * Np;
            double part = 0;
            for (int j = r0 + PG_TILE + lane; j < D; j += 32) part += Ri[j] * v.yb[j];
            part = warp_sum_d(part);
            if (lane == 0) rs[i] = (D < r0 + PG_TILE ? Rs[i][D - r0] : Ri[D]) - part;
        }
        __syncthreads();
        if (wid == 0)
            for (int i = nr - 1; i >= 0; i--) {
                double part = 0;
                for (int j = i + 1 + lane; j < nr; j += 32) part += Rs[i][j] * v.yb[r0 + j];
                part = warp_sum_d(part);
                if (lane == 0) v.yb[r0 + i] = (rs[i] - part) / Rs[i][i];
                __syncwarp();
            }
        __syncthreads();
    }
    chain_back_substitute(v, v.yb, Ls, Fn, xs, xn, rhs);
}

// ---- update: model cost change, candidate x [+] delta, its cost, the trust-region decision (sfm_bundle's order)
__global__ void __launch_bounds__(256) pg_update_kernel(PgLaunch a) {
    __shared__ double red[8];
    __shared__ int accept;
    const PgView v = pg_view(a, blockIdx.x);
    PgState* st = v.st;
    if (st->done) return;
    if (st->lin_fail) {  // invalid step: shrink the region like an unsuccessful one
        __syncthreads();
        if (threadIdx.x == 0) {
            st->iter++;
            st->lin_fail = 0;
            st->radius /= st->decrease;
            st->decrease *= 2;
            if (st->radius < 1e-32) st->done = 1;
        }
        return;
    }
    double step2 = 0, xn2 = 0;
    for (int k = threadIdx.x; k < v.n; k += blockDim.x) {
        const double* x = v.x + 4 * k;
        double* xc = v.xc + 4 * k;
        if (k < v.nc) {
            for (int p = 0; p < 4; p++) xc[p] = x[p];
            continue;
        }
        const double* d = v.dx + 4 * k;
        xc[0] = normalize_angle(x[0] + d[0]);
        for (int p = 1; p < 4; p++) xc[p] = x[p] + d[p];
        for (int p = 0; p < 4; p++) {
            step2 += d[p] * d[p];
            xn2 += x[p] * x[p];
        }
    }
    __syncthreads();
    double mc = 0, cc = 0;
    for (int k = threadIdx.x; k < v.n; k += blockDim.x)
        for (int e = 0; e < 5; e++) {
            const int b = edge_older(v, k, e);
            if (b < 0) continue;
            double r[4], J[32], rc[4];
            edge_eval(v, v.x, k, e, b, r, J);
            const double* di = v.dx + 4 * b;
            const double* dj = v.dx + 4 * k;
            const bool fi = b >= v.nc;
            for (int t = 0; t < 4; t++) {
                double jd = 0;
                for (int p = 0; p < 4; p++) jd += (fi ? J[8 * t + p] * di[p] : 0.0) + J[8 * t + 4 + p] * dj[p];
                mc -= jd * (r[t] + 0.5 * jd);
            }
            cc += edge_eval(v, v.xc, k, e, b, rc, nullptr);
        }
    mc = block_sum_d(mc, red);
    cc = block_sum_d(cc, red);
    step2 = block_sum_d(step2, red);
    xn2 = block_sum_d(xn2, red);
    if (threadIdx.x == 0) {
        int acc = 0;
        st->iter++;
        st->model_change = mc;
        st->cost_c = cc;
        if (!(mc > 0.0) || !isfinite(mc)) {
            st->radius /= st->decrease;
            st->decrease *= 2;
            if (st->radius < 1e-32) st->done = 1;
        } else if (sqrt(step2) <= 1e-8 * (sqrt(xn2) + 1e-8)) {  // parameter tolerance
            st->done = st->converged = 1;
        } else {
            const double change = st->cost - cc;
            if (isfinite(cc) && fabs(change) <= 1e-6 * st->cost) {  // function tolerance
                acc = change > 0.0;
                st->done = st->converged = 1;
            } else {
                const double rho = change / mc;
                if (isfinite(cc) && rho > 1e-3) {
                    acc = 1;
                    const double t = 2.0 * rho - 1.0;
                    st->radius = fmin(1e16, st->radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
                    st->decrease = 2.0;
                    st->need_lin = 1;
                } else {
                    st->radius /= st->decrease;
                    st->decrease *= 2;
                    if (st->radius < 1e-32) st->done = 1;
                }
            }
        }
        if (acc) {
            st->cost = cc;
            st->successful++;
        }
        accept = acc;
    }
    __syncthreads();
    if (accept)
        for (int i = threadIdx.x; i < 4 * v.n; i += blockDim.x) v.x[i] = v.xc[i];
}

__global__ void __launch_bounds__(256) pg_finish_kernel(PgLaunch a) {
    const PgView v = pg_view(a, blockIdx.x);
    for (int i = threadIdx.x; i < 4 * v.n; i += blockDim.x) v.out[i] = v.x[i];
    if (threadIdx.x == 0) {
        const PgState s = *v.st;
        double* o = v.out + pg_out_layout(v.n).summary;
        o[0] = s.iter; o[1] = s.successful; o[2] = s.cost0; o[3] = s.cost;
        o[4] = s.converged; o[5] = v.D; o[6] = v.n; o[7] = s.gmax;
    }
}

__global__ void pg_debug_edge_kernel(const double* prm, const double* meas, int weighted, int robust, double* out) {
    out[36] = four_dof_eval(prm, prm + 4, meas[4], meas[5], meas, weighted != 0, robust != 0, out, out + 4);
}

}  // namespace

int launch_pg_optimize(const PgLaunch& L, cudaStream_t s) {
    // pg_solve_kernel's dynamic shared memory (the Cholesky panel) is above the 48 KB default together with its static
    // part, and so is pg_panel_kernel's
    const size_t panel = sizeof(double) * CHOL_NB * CHOL_PS;
    if (raise_dynamic_smem((const void*)pg_solve_kernel, (int)panel) != cudaSuccess ||
        raise_dynamic_smem((const void*)pg_panel_kernel, (int)PG_PANEL_SMEM) != cudaSuccess)
        return -1;
    const int T = (std::min(L.max_D, PG_MAX_D) + 1 + 31) / 32;
    const int Tl = pg_tile_np(L.max_D) / PG_TILE;  // panels of the multi-CTA path, 0 when no member takes it
    const int chain_ctas = (L.max_D + 1 + 383) / 384;
    int launches = 0;
    pg_setup_kernel<<<L.count, 256, 0, s>>>(L);
    launches++;
    for (int it = 0; it < L.max_iterations; it++) {
        pg_linearize_kernel<<<L.count, 256, 0, s>>>(L);
        pg_chain_kernel<<<dim3(chain_ctas, L.count), 384, 0, s>>>(L);
        pg_border_kernel<<<dim3(T * (T + 1) / 2, L.count), 256, 0, s>>>(L);
        launches += 3;
        if (Tl) {
            pg_tile_kernel<false><<<dim3(Tl * (Tl + 1) / 2, L.count), 256, 0, s>>>(L, -1);
            launches++;
            for (int p = 0; p < Tl; p++) {
                pg_panel_kernel<<<dim3(Tl - p, L.count), 256, PG_PANEL_SMEM, s>>>(L, p);
                launches++;
                const int R = Tl - p - 1;
                if (R > 0) {
                    pg_tile_kernel<true><<<dim3(R * (R + 1) / 2, L.count), 256, 0, s>>>(L, p);
                    launches++;
                }
            }
        }
        pg_solve_kernel<<<L.count, 512, panel, s>>>(L);
        launches++;
        if (Tl) {
            pg_solve_large_kernel<<<L.count, 512, 0, s>>>(L);
            launches++;
        }
        pg_update_kernel<<<L.count, 256, 0, s>>>(L);
        launches++;
    }
    pg_finish_kernel<<<L.count, 256, 0, s>>>(L);
    return launches + 1;
}

void launch_pg_debug_edge(const double* d_params8, const double* d_meas6, int weighted, int robust, double* d_out, cudaStream_t s) {
    pg_debug_edge_kernel<<<1, 1, 0, s>>>(d_params8, d_meas6, weighted, robust, d_out);
}

}  // namespace vb
