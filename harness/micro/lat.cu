// Latency microbenchmarks (dependent chains, one warp) used to size the serial sections of the single-CTA solvers.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o harness/micro/lat harness/micro/lat.cu ; run on an H100.
#include <cstdio>
#include <cuda_runtime.h>
#define N 2048
template <int OP>
__global__ void chain(double x0, double* out, long long* clk) {
    __shared__ double sm[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sm[i] = 1.0 + 1e-9 * i;
    __syncthreads();
    double x = x0 + threadIdx.x * 1e-9, y = 1.000000001;
    long long t0 = clock64();
#pragma unroll 8
    for (int i = 0; i < N; i++) {
        if (OP == 0) x = fma(x, y, 1e-9);
        if (OP == 1) x = rsqrt(x) + 1.0;
        if (OP == 2) x = 1.0 / x + 0.5;
        if (OP == 3) x = sqrt(x) + 1.0;
        if (OP == 4) x = __shfl_xor_sync(0xffffffffu, x, 1);
        if (OP == 5) x = sm[((int)__double2int_rn(x)) & 255];
        if (OP == 6) x = x / y;
        if (OP == 7) x = (double)rsqrtf((float)x) + 1.0;
        if (OP == 8) x = __drcp_rn(x) + 0.5;
        if (OP == 9) x = x * y;
        if (OP == 10) x = x + y;
        if (OP == 11) x = hypot(x, y);
        if (OP == 12) { sm[threadIdx.x] = x; __syncwarp(); x = sm[threadIdx.x ^ 1]; }
        if (OP == 13) { sm[threadIdx.x & 255] = x; __syncthreads(); x = sm[(threadIdx.x ^ 1) & 255]; }
        if (OP == 14) { float f = (float)x; f = rsqrtf(f); x = (double)f + 1.0; }
        if (OP == 15) { float f = __double2float_rn(x); x = (double)(f * 1.0001f); }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) { out[OP] = x; clk[OP] = t1 - t0; }
}
int main() {
    double* d; long long* c;
    cudaMalloc(&d, 64 * 8); cudaMalloc(&c, 64 * 8);
    cudaMemset(c, 0, 64 * 8);
    const char* names[] = {"dfma", "rsqrt(double)+add", "1.0/x+add", "sqrt+add", "shfl double", "lds dependent (cvt+lds)", "x/y", "rsqrtf cvt+add", "__drcp_rn+add", "dmul", "dadd", "hypot", "sts+syncwarp+lds", "sts+syncthreads(512)+lds", "cvt/rsqrtf/cvt+add", "cvt f64->f32->f64"};
#define RUN(OP, T) chain<OP><<<1, T>>>(2.0, d, c);
    RUN(0, 32) RUN(1, 32) RUN(2, 32) RUN(3, 32) RUN(4, 32) RUN(5, 32) RUN(6, 32) RUN(7, 32) RUN(8, 32) RUN(9, 32) RUN(10, 32) RUN(11, 32) RUN(12, 32) RUN(13, 512) RUN(14, 32) RUN(15, 32)
    cudaDeviceSynchronize();
    long long h[64];
    cudaMemcpy(h, c, 64 * 8, cudaMemcpyDeviceToHost);
    for (int i = 0; i < 16; i++) printf("%-28s %7.1f cycles/op\n", names[i], (double)h[i] / N);
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
