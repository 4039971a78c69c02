// Every operation of vins_mono_b200/csrc/rotation.h behind one flat entry point, for tests/test_rotation_cpu.py (g++ with
// -ffp-contract=off) and tests/test_rotation_gpu.py (nvcc -x cu with --fmad=false, the same operations in a kernel).
// rot_eval(op, n, in, out) applies operation op to n records of ROT_IN[op] doubles and writes ROT_OUT[op] doubles each.
// Quaternions are (w, x, y, z), matrices row-major.
#include "rotation.h"

using namespace vb;

namespace {

enum { OP_R2YPR, OP_YPR2R, OP_QR, OP_FROMR, OP_NORMALIZE_ANGLE, OP_QMUL, OP_QROT, OP_MMUL, OP_MV, OP_NORMALIZED, OP_SKEW,
       OP_CROSS, OP_DOT, OP_QINV, OP_DELTAQ, OP_MT, OP_RODRIGUES, OP_COUNT };
constexpr int ROT_IN[OP_COUNT] = {9, 3, 4, 9, 1, 8, 7, 18, 12, 4, 3, 6, 6, 4, 3, 9, 3};
constexpr int ROT_OUT[OP_COUNT] = {3, 9, 9, 4, 1, 4, 3, 9, 3, 4, 9, 3, 1, 4, 4, 9, 9};

ROT_FN Vec3 v3(const double* p) { return Vec3(p[0], p[1], p[2]); }
ROT_FN Quat q4(const double* p) { return Quat(p[0], p[1], p[2], p[3]); }
ROT_FN Mat3 m9(const double* p) {
    Mat3 m;
    for (int i = 0; i < 9; i++) m.m[i] = p[i];
    return m;
}
ROT_FN void put(const Vec3& v, double* o) { o[0] = v.x; o[1] = v.y; o[2] = v.z; }
ROT_FN void put(const Quat& q, double* o) { o[0] = q.w; o[1] = q.x; o[2] = q.y; o[3] = q.z; }
ROT_FN void put(const Mat3& m, double* o) { for (int i = 0; i < 9; i++) o[i] = m.m[i]; }

ROT_FN void eval_one(int op, const double* in, double* o) {
    switch (op) {
        case OP_R2YPR: put(R2ypr(m9(in)), o); break;
        case OP_YPR2R: put(ypr2R(v3(in)), o); break;
        case OP_QR: put(q4(in).R(), o); break;
        case OP_FROMR: put(Quat::FromR(m9(in)), o); break;
        case OP_NORMALIZE_ANGLE: o[0] = normalize_angle(in[0]); break;
        case OP_QMUL: put(qmul(q4(in), q4(in + 4)), o); break;
        case OP_QROT: put(qrot(q4(in), v3(in + 4)), o); break;
        case OP_MMUL: put(m9(in) * m9(in + 9), o); break;
        case OP_MV: put(m9(in) * v3(in + 9), o); break;
        case OP_NORMALIZED: put(q4(in).normalized(), o); break;
        case OP_SKEW: put(skew(v3(in)), o); break;
        case OP_CROSS: put(cross(v3(in), v3(in + 3)), o); break;
        case OP_DOT: o[0] = dot(v3(in), v3(in + 3)); break;
        case OP_QINV: put(qinv(q4(in)), o); break;
        case OP_DELTAQ: put(deltaQ(v3(in)), o); break;
        case OP_MT: put(m9(in).T(), o); break;
        case OP_RODRIGUES: put(rodrigues(v3(in)), o); break;
    }
}

}  // namespace

extern "C" int rot_op_count() { return OP_COUNT; }
extern "C" int rot_op_width(int op, int out) { return op < 0 || op >= OP_COUNT ? -1 : out ? ROT_OUT[op] : ROT_IN[op]; }

extern "C" void rot_eval(int op, int n, const double* in, double* out) {
    for (int k = 0; k < n; k++) eval_one(op, in + (size_t)k * ROT_IN[op], out + (size_t)k * ROT_OUT[op]);
}

#ifdef __CUDACC__
namespace {
__global__ void rot_eval_kernel(int op, int n, int wi, int wo, const double* in, double* out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) eval_one(op, in + (size_t)k * wi, out + (size_t)k * wo);
}
}  // namespace

// The same records through the kernel; returns the CUDA error code.
extern "C" int rot_eval_device(int op, int n, const double* in, double* out) {
    const size_t bi = sizeof(double) * n * ROT_IN[op], bo = sizeof(double) * n * ROT_OUT[op];
    double *d_in = nullptr, *d_out = nullptr;
    cudaError_t e = cudaMalloc(&d_in, bi);
    if (e == cudaSuccess) e = cudaMalloc(&d_out, bo);
    if (e == cudaSuccess) e = cudaMemcpy(d_in, in, bi, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        rot_eval_kernel<<<(n + 127) / 128, 128>>>(op, n, ROT_IN[op], ROT_OUT[op], d_in, d_out);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, bo, cudaMemcpyDeviceToHost);
    cudaFree(d_in);
    cudaFree(d_out);
    return (int)e;
}
#endif
