// Phase timing of the single-CTA symmetric eigen-solver (vins_mono_b200/csrc/sym_eig.h) on a real marginalisation
// prior (harness/micro/prior75.bin: the 75x75 Schur complement A' of a steady-state frame, dumped from the CPU twin).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o harness/micro/eig_bench harness/micro/eig_bench.cu
#define SE_PROF 1
#include "../../vins_mono_b200/csrc/prior_floor.h"
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cmath>
using namespace vb;

__global__ void __launch_bounds__(512) eig_bench_kernel(const double* A, int n, int reps, double* evals, double* evecs, long long* clk) {
    extern __shared__ double V[];
    __shared__ double d[96], e[96], cs[4 * 96], scal[16];
    const int ld = n | 1;
    if (threadIdx.x < 16) se_clk[threadIdx.x] = 0;
    long long tot = 0;
    for (int r = 0; r < reps; r++) {
        for (int idx = threadIdx.x; idx < n * n; idx += blockDim.x) V[(idx / n) * ld + idx % n] = A[idx];
        __syncthreads();
        const long long t0 = clock64();
        sym_eig(CtaCtx(), V, n, ld, d, e, cs, scal);
        tot += clock64() - t0;
        __syncthreads();
    }
    for (int idx = threadIdx.x; idx < n * n; idx += blockDim.x) evecs[idx] = V[(idx / n) * ld + idx % n];
    for (int i = threadIdx.x; i < n; i += blockDim.x) evals[i] = d[i];
    if (threadIdx.x == 0) {
        for (int k = 0; k < 16; k++) clk[k] = se_clk[k] / reps;
        clk[16] = tot / reps;
        clk[17] = (long long)scal[4];
        clk[18] = (long long)scal[5];
    }
}

// The eps floor of the prior (prior_floor.h) on the same matrix: partial route (explicit eigenpairs below tau only) against the
// full decomposition.  Ain/gin are restored before every repetition; out: A+ | g0 | c0.
__global__ void __launch_bounds__(512) floor_bench_kernel(const double* Ain, const double* gin, int n, int reps, int partial, double* Ap,
                                                          double* g, double* c0, long long* clk, int* stats) {
    extern __shared__ double sm[];
    __shared__ double d[96], e[96], cs[4 * 96], scal[16], tv[96];
    const int ld = n | 1, nw = prior_floor_work(n, blockDim.x, 32);
    double* work = sm;
    double* V = sm + nw;
    if (threadIdx.x < 16) se_clk[threadIdx.x] = 0;
    long long tot = 0;
    for (int r = 0; r < reps; r++) {
        for (int idx = threadIdx.x; idx < n * n; idx += blockDim.x) Ap[idx] = Ain[idx];
        for (int i = threadIdx.x; i < n; i += blockDim.x) g[i] = gin[i];
        __syncthreads();
        const long long t0 = clock64();
        prior_floor<CtaCtx, 3>(CtaCtx(), Ap, g, c0, n, 1e-8, V, ld, d, e, cs, scal, tv, partial ? work : nullptr, work, stats);
        tot += clock64() - t0;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        for (int k = 0; k < 16; k++) clk[k] = se_clk[k] / reps;
        clk[16] = tot / reps;
    }
}

int main(int argc, char** argv) {
    const int n = 75, reps = 5;
    std::vector<double> A(n * n);
    FILE* f = fopen(argc > 1 ? argv[1] : "harness/micro/prior75.bin", "rb");
    if (!f || fread(A.data(), 8, n * n, f) != (size_t)n * n) { printf("cannot read prior\n"); return 1; }
    fclose(f);
    double *dA, *dw, *dV; long long* dclk;
    cudaMalloc(&dA, n * n * 8); cudaMalloc(&dw, n * 8); cudaMalloc(&dV, n * n * 8); cudaMalloc(&dclk, 32 * 8);
    cudaMemcpy(dA, A.data(), n * n * 8, cudaMemcpyHostToDevice);
    const int smem = n * (n | 1) * 8 + 64;
    cudaFuncSetAttribute(eig_bench_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    for (int threads : {512, 256, 128}) {
        eig_bench_kernel<<<1, threads, smem>>>(dA, n, reps, dw, dV, dclk);
        cudaDeviceSynchronize();
        std::vector<double> w(n), V(n * n); long long clk[32];
        cudaMemcpy(w.data(), dw, n * 8, cudaMemcpyDeviceToHost);
        cudaMemcpy(V.data(), dV, n * n * 8, cudaMemcpyDeviceToHost);
        cudaMemcpy(clk, dclk, 32 * 8, cudaMemcpyDeviceToHost);
        double res = 0, amax = 0, orth = 0;
        for (int i = 0; i < n; i++) for (int k = 0; k < n; k++) {
            double s = 0, o = 0;
            for (int j = 0; j < n; j++) { s += A[i * n + j] * V[j * n + k]; o += V[j * n + i] * V[j * n + k]; }
            res = fmax(res, fabs(s - V[i * n + k] * w[k])); amax = fmax(amax, fabs(A[i * n + k])); orth = fmax(orth, fabs(o - (i == k)));
        }
        printf("threads %d: %s  |AV-VW|/|A| = %.2e  |VtV-I| = %.2e   total %lld cycles (tridiag %lld, QL %lld)\n", threads,
               cudaGetErrorString(cudaGetLastError()), res / amax, orth, clk[16], clk[17], clk[18]);
        const char* names[] = {"tred2 A: matvec || |u|^2, scalars", "tred2 B: fix, scale, p -= f/2h u", "tred2 C: rank-2 update, next u", "(unused)", "(unused)",
                               "(unused)", "accum dots", "accum update + zero column", "QL search/bookkeeping", "QL wait for consumers", "QL sweep recurrence"};
        for (int k = 0; k < 11; k++) printf("    %-34s %9lld\n", names[k], clk[k]);
    }
    {   // prior floor: both routes
        std::vector<double> g(n);
        unsigned sd = 99;
        std::vector<double> r(n);
        for (auto& v : r) { sd = sd * 1664525u + 1013904223u; v = ((sd >> 8) & 0xffff) / 65536.0 - 0.5; }
        for (int i = 0; i < n; i++) { double s = 0; for (int j = 0; j < n; j++) s += 0.5 * (A[i * n + j] + A[j * n + i]) * r[j]; g[i] = s; }  // b' in the range of A'
        double *dg, *dAp, *dgo, *dc; int* dst;
        cudaMalloc(&dg, n * 8); cudaMalloc(&dAp, n * n * 8); cudaMalloc(&dgo, n * 8); cudaMalloc(&dc, 8); cudaMalloc(&dst, 8);
        cudaMemcpy(dg, g.data(), n * 8, cudaMemcpyHostToDevice);
        const int fsm = (prior_floor_work(n, 512, 32) + n * (n | 1)) * 8 + 64;
        cudaFuncSetAttribute(floor_bench_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, fsm);
        std::vector<double> Aout[2], gout[2]; double c0[2]; int st[2][2];
        for (int partial = 0; partial < 2; partial++) {
            floor_bench_kernel<<<1, 512, fsm>>>(dA, dg, n, reps, partial, dAp, dgo, dc, dclk, dst);
            cudaDeviceSynchronize();
            long long clk[32];
            Aout[partial].resize(n * n); gout[partial].resize(n);
            cudaMemcpy(Aout[partial].data(), dAp, n * n * 8, cudaMemcpyDeviceToHost);
            cudaMemcpy(gout[partial].data(), dgo, n * 8, cudaMemcpyDeviceToHost);
            cudaMemcpy(&c0[partial], dc, 8, cudaMemcpyDeviceToHost);
            cudaMemcpy(st[partial], dst, 8, cudaMemcpyDeviceToHost);
            cudaMemcpy(clk, dclk, 32 * 8, cudaMemcpyDeviceToHost);
            printf("prior floor, %s: %s  explicit pairs %d dropped %d  c0 %.12g  total %lld cycles\n", partial ? "partial route" : "full decomposition",
                   cudaGetErrorString(cudaGetLastError()), st[partial][0], st[partial][1], c0[partial], clk[16]);
            if (partial) {
                const char* nm[] = {"bisection", "inverse iteration + MGS", "Rayleigh q. + back-transformation", "A+, g0, M, LDL^T"};
                printf("    tridiagonalisation A/B/C           %9lld\n", clk[0] + clk[1] + clk[2]);
                for (int k = 0; k < 4; k++) printf("    %-34s %9lld\n", nm[k], clk[11 + k]);
            }
        }
        double dAm = 0, am = 0, dgm = 0, gm = 0;
        for (int i = 0; i < n * n; i++) { dAm = fmax(dAm, fabs(Aout[0][i] - Aout[1][i])); am = fmax(am, fabs(Aout[0][i])); }
        for (int i = 0; i < n; i++) { dgm = fmax(dgm, fabs(gout[0][i] - gout[1][i])); gm = fmax(gm, fabs(gout[0][i])); }
        printf("routes agree: |dA+|/|A+| = %.2e  |dg0|/|g0| = %.2e  dc0/c0 = %.2e\n", dAm / am, dgm / gm, fabs(c0[0] - c0[1]) / c0[0]);
    }
    return 0;
}
