// Phase timing of the single-CTA packed Cholesky / triangular solves of ba_step_kernel on a synthetic SPD matrix.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I include -I vins_mono_b200/csrc -o harness/micro/chol_bench harness/micro/chol_bench.cu
#define CHOL_PROF 1
#include "../../vins_mono_b200/csrc/ba_kernels.cu"
#include <cstdio>
#include <vector>
#include <cmath>
using namespace vb;

__global__ void __launch_bounds__(512) chol_bench_kernel(const double* Ain, int n, int reps, double* Lout, long long* clk, int mode) {
    extern __shared__ __align__(16) double dyn[];
    double* Pc = dyn;
    double* Lp = dyn + CHOL_NB * CHOL_PS;
    __shared__ double rdiag[BA_MAX_D], linv[(BA_MAX_D / CHOL_NB) * 64], y[BA_MAX_D];
    __shared__ int flag;
    const int np = n * (n + 1) / 2;
    if (threadIdx.x < 8) chol_clk[threadIdx.x] = 0;
    long long total = 0, tsolve = 0;
    for (int r = 0; r < reps; r++) {
        for (int i = threadIdx.x; i < np; i += blockDim.x) Lp[i] = Ain[i];
        for (int i = threadIdx.x; i <= n; i += blockDim.x) Lp[np + i] = i < n ? 1.0 + i : 0.0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = 1.0 + i;
        __syncthreads();
        const long long t0 = clock64();
        cholesky_packed(Lp, Pc, n, rdiag, linv, &flag, n + 1);
        const long long t1 = clock64();
        if (mode) {
            for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = Lp[np + i];
            __syncthreads();
            chol_solve_packed(Lp, linv, n, y, false);
        }
        __syncthreads();
        const long long t2 = clock64();
        total += t1 - t0;
        tsolve += t2 - t1;
    }
    for (int i = threadIdx.x; i < np; i += blockDim.x) Lout[i] = Lp[i];
    for (int i = threadIdx.x; i < n; i += blockDim.x) Lout[np + i] = y[i];
    if (threadIdx.x == 0) {
        for (int k = 0; k < 8; k++) clk[k] = chol_clk[k] / reps;
        clk[8] = total / reps;
        clk[9] = tsolve / reps;
        clk[10] = flag;
    }
}

int main(int argc, char** argv) {
    const int n = argc > 1 ? atoi(argv[1]) : 172, reps = 10;
    const int np = n * (n + 1) / 2;
    std::vector<double> B(n * n), A(n * n, 0.0), Ap(np);
    unsigned s = 12345;
    for (auto& v : B) { s = s * 1664525u + 1013904223u; v = ((s >> 8) & 0xffff) / 65536.0 - 0.5; }
    for (int i = 0; i < n; i++) for (int j = 0; j <= i; j++) {
        double acc = i == j ? 1.0 : 0.0;
        for (int k = 0; k < n; k++) acc += B[i * n + k] * B[j * n + k];
        A[i * n + j] = A[j * n + i] = acc;
        Ap[i * (i + 1) / 2 + j] = acc;
    }
    // host Cholesky for checking
    std::vector<double> L(A);
    for (int j = 0; j < n; j++) {
        for (int k = 0; k < j; k++) for (int i = j; i < n; i++) L[i * n + j] -= L[i * n + k] * L[j * n + k];
        const double d = std::sqrt(L[j * n + j]);
        for (int i = j; i < n; i++) L[i * n + j] /= d;
    }
    double *dA, *dL; long long* dclk;
    cudaMalloc(&dA, np * 8); cudaMalloc(&dL, (np + n) * 8); cudaMalloc(&dclk, 16 * 8);
    cudaMemcpy(dA, Ap.data(), np * 8, cudaMemcpyHostToDevice);
    const int dynb = (np + n + 1 + CHOL_NB * CHOL_PS) * 8;
    cudaFuncSetAttribute(chol_bench_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dynb);
    chol_bench_kernel<<<1, 512, dynb>>>(dA, n, reps, dL, dclk, 1);
    cudaDeviceSynchronize();
    printf("launch: %s\n", cudaGetErrorString(cudaGetLastError()));
    std::vector<double> Lg(np + n); long long clk[16];
    cudaMemcpy(Lg.data(), dL, (np + n) * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(clk, dclk, 16 * 8, cudaMemcpyDeviceToHost);
    double err = 0;
    for (int i = 0; i < n; i++) for (int j = 0; j <= i; j++) err = fmax(err, fabs(Lg[i * (i + 1) / 2 + j] - L[i * n + j]));
    // reference solution of A y = b, b_i = 1 + i
    std::vector<double> yr(n);
    for (int i = 0; i < n; i++) { double v = 1.0 + i; for (int k = 0; k < i; k++) v -= L[i * n + k] * yr[k]; yr[i] = v / L[i * n + i]; }
    for (int i = n - 1; i >= 0; i--) { double v = yr[i]; for (int k = i + 1; k < n; k++) v -= L[k * n + i] * yr[k]; yr[i] = v / L[i * n + i]; }
    double yerr = 0, ymax = 0;
    for (int i = 0; i < n; i++) { yerr = fmax(yerr, fabs(Lg[np + i] - yr[i])); ymax = fmax(ymax, fabs(yr[i])); }
    printf("n=%d ok=%lld max|L-Lref|=%.3e  max|y-yref|/|y|=%.3e\n", n, clk[10], err, yerr / ymax);
    const char* names[] = {"diag: load+update", "diag: factor chain", "diag: store", "loop top", "panel", "sync after panel", "warp0 diag total/others tiles", "sync after trailing"};
    for (int k = 0; k < 8; k++) printf("  %-34s %9lld cycles\n", names[k], clk[k]);
    printf("  cholesky total %lld, solve total %lld cycles\n", clk[8], clk[9]);
    return 0;
}
