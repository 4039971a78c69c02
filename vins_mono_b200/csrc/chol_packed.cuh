// Packed dense Cholesky of the device solvers (one CTA per system): ba_kernels.cu factorises the BA step's reduced
// system with it, pg_kernels.cu the pose graph's border system.  Included at file scope; everything is internal to
// the including translation unit.
#pragma once

namespace vb {
namespace {

// In-place lower Cholesky of the n x n matrix stored packed (row-major lower triangle) in `Lp`; rdiag receives
// 1 / L_kk, linv the inverses of the 8x8 diagonal blocks (for the triangular solves).  Right-looking, blocked by 8
// columns, with one block of look-ahead: the trailing update is split into the next block column (all warps, "part A")
// and the rest ("part B"); warp 0 factorises the next 8x8 diagonal block in registers (one row per lane, pivots and
// multipliers exchanged with shuffles) WHILE the other warps run part B, which takes the serial diagonal chain
// (8 dependent rsqrt + shuffle rounds) off the critical path.  The panel below a diagonal block is solved by one
// thread per row, trailing tiles are 4x4 register tiles (0.5 shared-memory loads per FMA).  3 barriers per block column.
#define CHOL_NB 8
#define CHOL_PS 360  // panel copy stride: BA_MAX_D + 8 rows of slack for partial tiles
#ifdef CHOL_PROF  // harness/micro/chol_bench.cu: per-phase cycle counters kept in shared memory by thread 0
__shared__ long long chol_clk[8];
#define CP_BEGIN() long long cp0_ = clock64()
#define CP(k) do { if (threadIdx.x == 0) { const long long c1_ = clock64(); chol_clk[k] += c1_ - cp0_; cp0_ = c1_; } } while (0)
#else
#define CP_BEGIN() do {} while (0)
#define CP(k) do {} while (0)
#endif
// One full warp factorises the diagonal block starting at kb (w columns) and publishes it in dblk and rdiag.
// When upd != 0 the pending rank-8 update from the previous panel (held column-major in Pc) is applied first: the 64
// entries of the block are spread over the lanes (a length-8 dot product each) and staged in shared memory.  Every
// lane then factorises the WHOLE 8x8 block redundantly in registers: no shuffles, so the dependent chain per column
// is rsqrt -> scale -> one FMA (one row per lane with shuffled pivots/multipliers measured 2.6k cycles per block for
// the chain alone, this form 1.1k; harness/micro/chol_bench.cu).  Rows >= w behave like identity rows.
__device__ __forceinline__ void chol_diag_block(double* Lp, const double* Pc, int kb, int w, double* rdiag,
                                                double (*dblk)[CHOL_NB + 1], int* flag, int upd, double* stage, int nrows) {
    const int lane = threadIdx.x & 31;
    CP_BEGIN();
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int e = lane + 32 * h, rr = e >> 3, c = e & 7;
        double v = (rr == c) ? 1.0 : 0.0;
        if (rr < w && c <= rr) {
            v = Lp[(kb + rr) * (kb + rr + 1) / 2 + kb + c];
            if (upd) {
                double acc0 = 0.0, acc1 = 0.0;
#pragma unroll
                for (int t = 0; t < CHOL_NB; t += 2) {
                    acc0 += Pc[t * CHOL_PS + kb + rr] * Pc[t * CHOL_PS + kb + c];
                    acc1 += Pc[(t + 1) * CHOL_PS + kb + rr] * Pc[(t + 1) * CHOL_PS + kb + c];
                }
                v -= acc0 + acc1;
            }
        } else if (upd && rr >= w && kb + rr < nrows && c < w) {
            // a row below a partial last block (the appended right-hand-side row): it only receives the update
            double acc0 = 0.0;
#pragma unroll
            for (int t = 0; t < CHOL_NB; t++) acc0 += Pc[t * CHOL_PS + kb + rr] * Pc[t * CHOL_PS + kb + c];
            Lp[(kb + rr) * (kb + rr + 1) / 2 + kb + c] -= acc0;
        }
        stage[e] = v;
    }
    __syncwarp();
    double a[CHOL_NB][CHOL_NB];
#pragma unroll
    for (int rr = 0; rr < CHOL_NB; rr++)
#pragma unroll
        for (int c = 0; c <= rr; c++) a[rr][c] = stage[rr * CHOL_NB + c];
    CP(0);
    bool ok = true;
#pragma unroll
    for (int c = 0; c < CHOL_NB; c++) {
        const double piv = a[c][c];
        if (!(piv > 0.0) || !isfinite(piv)) ok = false;
        const double rc = rsqrt(piv);
        a[c][c] = piv * rc;
#pragma unroll
        for (int rr = c + 1; rr < CHOL_NB; rr++) a[rr][c] *= rc;
        // column c is final: every lane holds the same values and stores them to the same addresses of the small block
        // buffer (the stores fill the latency bubbles of the chain and free the registers early).  The copy into the
        // packed matrix is left to idle threads of the next panel phase: stores to the big array queue behind the tile
        // warps' traffic and cost this chain 30 k cycles per factorisation when issued here.
        if (c < w) {
            rdiag[kb + c] = rc;
#pragma unroll
            for (int rr = c; rr < CHOL_NB; rr++)
                if (rr < w) dblk[rr][c] = a[rr][c];
        }
#pragma unroll
        for (int k = c + 1; k < CHOL_NB; k++)
#pragma unroll
            for (int rr = k; rr < CHOL_NB; rr++) a[rr][k] -= a[rr][c] * a[k][c];
    }
    CP(1);
    if (!ok && lane == 0) *flag = 0;
    CP(2);
}

// Trailing update of one 8 (rows) x 4 (columns) register tile from the current panel.  The panel is read from its
// column-major copy Pc: a thread's 8 (4) consecutive rows of one panel column are 64 (32) contiguous bytes, so the
// loads are 128-bit, conflict-free across a warp (consecutive lanes = consecutive column tiles) and the row operand is
// a broadcast.  0.375 loads per FMA; the packed matrix is only touched for the final read-modify-write.
__device__ __forceinline__ void chol_tile84(double* Lp, const double* Pc, int n, int ke, int ti8, int tj4) {
    const int i0 = ke + 8 * ti8, j0 = ke + 4 * tj4;
    double acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int q = 0; q < 4; q++) acc[r][q] = 0.0;
#pragma unroll
    for (int c = 0; c < CHOL_NB; c++) {
        const double2* pi = reinterpret_cast<const double2*>(Pc + c * CHOL_PS + i0);
        const double2* pj = reinterpret_cast<const double2*>(Pc + c * CHOL_PS + j0);
        const double2 i01 = pi[0], i23 = pi[1], i45 = pi[2], i67 = pi[3];
        const double2 j01 = pj[0], j23 = pj[1];
        const double li[8] = {i01.x, i01.y, i23.x, i23.y, i45.x, i45.y, i67.x, i67.y};
        const double lj[4] = {j01.x, j01.y, j23.x, j23.y};
#pragma unroll
        for (int r = 0; r < 8; r++)
#pragma unroll
            for (int q = 0; q < 4; q++) acc[r][q] += li[r] * lj[q];
    }
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int i = i0 + r;
        if (i < n) {
            const int ib = i * (i + 1) / 2;
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (j0 + q <= i) Lp[ib + j0 + q] -= acc[r][q];
        }
    }
}

// Pc: CHOL_NB * CHOL_PS doubles of 16-byte aligned shared memory (current panel, column-major, rows >= n zero).
// nrows >= n: rows n .. nrows-1 of the packed array are carried along without being factorised (row n = a right-hand
// side b turns into L^-1 b, i.e. the forward substitution comes for free with the trailing updates).
__device__ bool cholesky_packed(double* Lp, double* Pc, int n, double* rdiag, double* linv, int* flag, int nrows) {
    __shared__ double dblk[CHOL_NB][CHOL_NB + 1], stage[CHOL_NB * CHOL_NB];
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) *flag = 1;
    for (int c = 0; c < CHOL_NB; c++)
        for (int i = nrows + tid; i < CHOL_PS; i += nt) Pc[c * CHOL_PS + i] = 0.0;
    __syncthreads();
    if (tid < 32) chol_diag_block(Lp, Pc, 0, min(CHOL_NB, n), rdiag, dblk, flag, 0, stage, nrows);
    __syncthreads();
    CP_BEGIN();
    for (int kb = 0; kb < n; kb += CHOL_NB) {
        const int w = min(CHOL_NB, n - kb), ke = kb + w;  // only the last block can be partial
        if (!*flag) return false;
        if (tid >= nt - 64) {  // factorised diagonal block -> packed matrix (threads that have no panel row)
            const int e = tid - (nt - 64), rr = e >> 3, c = e & 7;
            if (rr < w && c <= rr) Lp[(kb + rr) * (kb + rr + 1) / 2 + kb + c] = dblk[rr][c];
        }
        if (ke >= nrows) break;
        CP(3);
        // panel: rows below the diagonal block, forward substitution against it
        for (int i = ke + tid; i < nrows; i += nt) {
            double x[CHOL_NB];
            const int ib = i * (i + 1) / 2 + kb;
#pragma unroll
            for (int c = 0; c < CHOL_NB; c++) {
                double v = 0.0;
                if (c < w) {
                    v = Lp[ib + c];
#pragma unroll
                    for (int t = 0; t < c; t++) v -= x[t] * dblk[c][t];
                    v *= rdiag[kb + c];
                    Lp[ib + c] = v;
                }
                x[c] = v;
                Pc[c * CHOL_PS + i] = v;
            }
        }
        CP(4);
        __syncthreads();
        CP(5);
        if (ke >= n) break;  // nothing left to factorise (the carried rows are complete)
        // warp 0: next diagonal block (update + factorisation); the others: every other trailing tile.  Tile row
        // ti8 holds the column tiles tj4 = 0 .. 2 ti8 + 1 (t = ti8 (ti8 + 1) + tj4); t = 0, 1 are the diagonal block.
        if (tid < 32) {
            chol_diag_block(Lp, Pc, ke, min(CHOL_NB, n - ke), rdiag, dblk, flag, 1, stage, nrows);
        } else {
            const int m = nrows - ke, nr8 = (m + 7) / 8, ntiles = nr8 * (nr8 + 1);
            for (int t = 2 + tid - 32; t < ntiles; t += nt - 32) {
                int ti8 = (int)((sqrtf(4.f * (float)t + 1.f) - 1.f) * 0.5f);
                while (ti8 * (ti8 + 1) > t) ti8--;
                while ((ti8 + 1) * (ti8 + 2) <= t) ti8++;
                chol_tile84(Lp, Pc, nrows, ke, ti8, t - ti8 * (ti8 + 1));
            }
        }
        CP(6);
        __syncthreads();
        CP(7);
    }
    // inverses of the diagonal blocks (lower triangular), one block per warp, one column per lane: the triangular
    // solves then need an 8x8 product per block instead of a dependent substitution chain
    const int wid = tid >> 5, nw = nt >> 5, lane = tid & 31;
    for (int blk = wid; blk * CHOL_NB < n; blk += nw) {
        const int kb = blk * CHOL_NB, w = min(CHOL_NB, n - kb);
        if (lane < CHOL_NB) {
            const int c = lane;
            double x[CHOL_NB];
#pragma unroll
            for (int rr = 0; rr < CHOL_NB; rr++) {
                double v = 0.0;
                if (rr >= c && rr < w && c < w) {
                    v = (rr == c) ? 1.0 : 0.0;
                    const size_t rb = (size_t)(kb + rr) * (kb + rr + 1) / 2 + kb;
#pragma unroll
                    for (int k = 0; k < CHOL_NB; k++)
                        if (k >= c && k < rr) v -= Lp[rb + k] * x[k];
                    v *= rdiag[kb + rr];
                }
                x[rr] = v;
                linv[blk * 64 + rr * CHOL_NB + c] = v;
            }
        }
    }
    __syncthreads();
    return true;
}

// Solves L L^T y = b with the packed factor; y (in/out) in shared memory, all threads of the CTA take part.
// Blocked by 8: the 8x8 triangular block is applied through its precomputed inverse (8 lanes, independent dot
// products), the remaining rows are updated with 8 columns at once by one thread per row.
__device__ void chol_solve_packed(const double* Lp, const double* linv, int n, double* y, bool forward = true) {
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int kb = 0; forward && kb < n; kb += CHOL_NB) {  // forward: L z = b
        const int w = min(CHOL_NB, n - kb), ke = kb + w;
        if (tid < 32) {
            double v = 0.0;
            const double* Li = linv + (kb / CHOL_NB) * 64;
            if (tid < w)
                for (int c = 0; c <= tid; c++) v += Li[tid * CHOL_NB + c] * y[kb + c];
            __syncwarp();
            if (tid < w) y[kb + tid] = v;
        }
        __syncthreads();
        for (int i = ke + tid; i < n; i += nt) {
            const size_t ib = (size_t)i * (i + 1) / 2 + kb;
            double v = y[i];
#pragma unroll
            for (int c = 0; c < CHOL_NB; c++)
                if (c < w) v -= Lp[ib + c] * y[kb + c];
            y[i] = v;
        }
        __syncthreads();
    }
    const int last = ((n - 1) / CHOL_NB) * CHOL_NB;
    for (int kb = last; kb >= 0; kb -= CHOL_NB) {  // backward: L^T y = z
        const int w = min(CHOL_NB, n - kb);
        if (tid < 32) {
            double v = 0.0;
            const double* Li = linv + (kb / CHOL_NB) * 64;
            if (tid < w)
                for (int r = tid; r < w; r++) v += Li[r * CHOL_NB + tid] * y[kb + r];
            __syncwarp();
            if (tid < w) y[kb + tid] = v;
        }
        __syncthreads();
        for (int i = tid; i < kb; i += nt) {
            double v = y[i];
#pragma unroll
            for (int c = 0; c < CHOL_NB; c++)
                if (c < w) v -= Lp[(size_t)(kb + c) * (kb + c + 1) / 2 + i] * y[kb + c];
            y[i] = v;
        }
        __syncthreads();
    }
}

}  // namespace
}  // namespace vb
