// 3-vectors, 3x3 matrices and quaternions for host and device code alike: the Eigen arithmetic the reference uses and its
// Utility rotation helpers (utility.h:70-112, pose_graph.h:89-97), written once.  Eigen is not a dependency here.
// Every operation has one body.  Where host code spells one as a member (q.R(), A * B, A * v, A.T(), q.normalized()), the
// member forwards to the free function the device code calls.  Functions built from +, -, *, / and sqrt give the same
// doubles on host and device when both compile without FMA contraction (-ffp-contract=off, --fmad=false); R2ypr, ypr2R
// and rodrigues also call atan2, sin or cos, whose last bits differ between CUDA's math library and glibc.
// Vec3 defaults to zero, Mat3 and Quat to the identity; host code relies on these defaults.
#pragma once
#include <cmath>
#include <cstring>

#ifdef __CUDACC__
#define ROT_FN __host__ __device__ __forceinline__
#else
#define ROT_FN inline
#endif

namespace vb {

struct Vec3 {
    double x = 0, y = 0, z = 0;
    ROT_FN Vec3() {}
    ROT_FN Vec3(double a, double b, double c) : x(a), y(b), z(c) {}
    ROT_FN Vec3 operator+(const Vec3& o) const { return {x + o.x, y + o.y, z + o.z}; }
    ROT_FN Vec3 operator-(const Vec3& o) const { return {x - o.x, y - o.y, z - o.z}; }
    ROT_FN Vec3 operator*(double s) const { return {x * s, y * s, z * s}; }
    ROT_FN Vec3& operator+=(const Vec3& o) { x += o.x; y += o.y; z += o.z; return *this; }
    ROT_FN double norm() const { return sqrt(x * x + y * y + z * z); }
    ROT_FN double operator[](int i) const { return i == 0 ? x : i == 1 ? y : z; }
};
ROT_FN Vec3 operator*(double s, const Vec3& v) { return v * s; }

struct Mat3 {  // row-major
    double m[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    ROT_FN double& operator()(int i, int j) { return m[3 * i + j]; }
    ROT_FN double operator()(int i, int j) const { return m[3 * i + j]; }
    ROT_FN Mat3 operator*(const Mat3& o) const;
    ROT_FN Vec3 operator*(const Vec3& v) const;
    ROT_FN Mat3 T() const;
    ROT_FN Vec3 col(int j) const { return {m[j], m[3 + j], m[6 + j]}; }
};

struct Quat {
    double w = 1, x = 0, y = 0, z = 0;
    ROT_FN Quat() {}
    ROT_FN Quat(double w_, double x_, double y_, double z_) : w(w_), x(x_), y(y_), z(z_) {}
    ROT_FN Quat normalized() const;
    ROT_FN Mat3 R() const;
    static ROT_FN Quat FromR(const Mat3& m);  // Eigen's Quaterniond(Matrix3d), branch for branch
};

ROT_FN double dot(const Vec3& a, const Vec3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
ROT_FN Vec3 cross(const Vec3& a, const Vec3& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

ROT_FN Mat3 mmul(const Mat3& a, const Mat3& b) {
    Mat3 r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
    return r;
}
ROT_FN Mat3 mT(const Mat3& a) {
    Mat3 r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * j + i];
    return r;
}
ROT_FN Vec3 mv(const Mat3& a, const Vec3& v) {
    return {a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z, a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z, a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z};
}
ROT_FN Mat3 skew(const Vec3& q) {
    Mat3 r;
    r.m[0] = 0;    r.m[1] = -q.z; r.m[2] = q.y;
    r.m[3] = q.z;  r.m[4] = 0;    r.m[5] = -q.x;
    r.m[6] = -q.y; r.m[7] = q.x;  r.m[8] = 0;
    return r;
}
ROT_FN Mat3 mscale(const Mat3& a, double s) { Mat3 r; for (int i = 0; i < 9; i++) r.m[i] = a.m[i] * s; return r; }
ROT_FN Mat3 madd(const Mat3& a, const Mat3& b) { Mat3 r; for (int i = 0; i < 9; i++) r.m[i] = a.m[i] + b.m[i]; return r; }
ROT_FN Mat3 msub(const Mat3& a, const Mat3& b) { Mat3 r; for (int i = 0; i < 9; i++) r.m[i] = a.m[i] - b.m[i]; return r; }

ROT_FN Mat3 Mat3::operator*(const Mat3& o) const { return mmul(*this, o); }
ROT_FN Vec3 Mat3::operator*(const Vec3& v) const { return mv(*this, v); }
ROT_FN Mat3 Mat3::T() const { return mT(*this); }

// Eigen's quaternion product
ROT_FN Quat qmul(const Quat& a, const Quat& b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
ROT_FN Quat qinv(const Quat& q) {
    const double n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
}
ROT_FN Quat qnormalized(const Quat& q) {
    const double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    return {q.w / n, q.x / n, q.y / n, q.z / n};
}
ROT_FN Vec3 qrot(const Quat& q, const Vec3& v) {  // Eigen's quaternion * vector
    const Vec3 u(q.x, q.y, q.z);
    Vec3 uv = cross(u, v);
    uv = uv + uv;
    return v + q.w * uv + cross(u, uv);
}
ROT_FN Mat3 qR(const Quat& q) {  // Eigen's toRotationMatrix
    Mat3 r;
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    r.m[0] = 1 - (tyy + tzz); r.m[1] = txy - twz;       r.m[2] = txz + twy;
    r.m[3] = txy + twz;       r.m[4] = 1 - (txx + tzz); r.m[5] = tyz - twx;
    r.m[6] = txz - twy;       r.m[7] = tyz + twx;       r.m[8] = 1 - (txx + tyy);
    return r;
}
// Utility::deltaQ, not normalised
ROT_FN Quat deltaQ(const Vec3& th) { return {1.0, th.x / 2.0, th.y / 2.0, th.z / 2.0}; }

ROT_FN Quat Quat::normalized() const { return qnormalized(*this); }
ROT_FN Mat3 Quat::R() const { return qR(*this); }
ROT_FN Quat Quat::FromR(const Mat3& m) {
    Quat q;
    double t = m(0, 0) + m(1, 1) + m(2, 2);
    if (t > 0) {
        t = sqrt(t + 1.0);
        q.w = 0.5 * t;
        t = 0.5 / t;
        q.x = (m(2, 1) - m(1, 2)) * t;
        q.y = (m(0, 2) - m(2, 0)) * t;
        q.z = (m(1, 0) - m(0, 1)) * t;
    } else {
        int i = 0;
        if (m(1, 1) > m(0, 0)) i = 1;
        if (m(2, 2) > m(i, i)) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
        double c[3];
        c[i] = 0.5 * t;
        t = 0.5 / t;
        q.w = (m(k, j) - m(j, k)) * t;
        c[j] = (m(j, i) + m(i, j)) * t;
        c[k] = (m(k, i) + m(i, k)) * t;
        q.x = c[0]; q.y = c[1]; q.z = c[2];
    }
    return q;
}

// Utility::R2ypr (utility.h:70-85): yaw, pitch, roll in degrees
ROT_FN Vec3 R2ypr(const Mat3& R) {
    const Vec3 n = R.col(0), o = R.col(1), a = R.col(2);
    const double y = atan2(n.y, n.x);
    const double p = atan2(-n.z, n.x * cos(y) + n.y * sin(y));
    const double r = atan2(a.x * sin(y) - a.y * cos(y), -o.x * sin(y) + o.y * cos(y));
    return Vec3(y, p, r) * (1.0 / M_PI * 180.0);
}
// Utility::ypr2R (utility.h:88-112)
ROT_FN Mat3 ypr2R(const Vec3& ypr) {
    const double y = ypr.x / 180.0 * M_PI, p = ypr.y / 180.0 * M_PI, r = ypr.z / 180.0 * M_PI;
    Mat3 Rz, Ry, Rx;
    Rz(0, 0) = cos(y); Rz(0, 1) = -sin(y); Rz(1, 0) = sin(y); Rz(1, 1) = cos(y);
    Ry(0, 0) = cos(p); Ry(0, 2) = sin(p); Ry(2, 0) = -sin(p); Ry(2, 2) = cos(p);
    Rx(1, 1) = cos(r); Rx(1, 2) = -sin(r); Rx(2, 1) = sin(r); Rx(2, 2) = cos(r);
    return Rz * Ry * Rx;
}
// Utility::normalizeAngle / NormalizeAngle (pose_graph.h:89-97), degrees
ROT_FN double normalize_angle(double a) {
    if (a > 180.0) return a - 360.0;
    if (a < -180.0) return a + 360.0;
    return a;
}
// Rodrigues: the rotation matrix of the rotation vector w; below |w| = 1e-12, I + [w]x + [w]x^2 / 2
ROT_FN Mat3 rodrigues(const Vec3& w) {
    const double th = w.norm();
    const double a = th < 1e-12 ? 1.0 : sin(th) / th, b = th < 1e-12 ? 0.5 : (1.0 - cos(th)) / (th * th);
    const Mat3 K = skew(w), K2 = K * K;
    Mat3 R;
    for (int i = 0; i < 9; i++) R.m[i] = (i % 4 == 0 ? 1.0 : 0.0) + a * K.m[i] + b * K2.m[i];
    return R;
}

// Direction of the smallest singular value of a (rows x 4) matrix: one-sided Jacobi on its columns.  Host only.
inline void null_direction4(const double* A, int rows, double v[4]) {
    double U[64 * 4], V[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    std::memcpy(U, A, sizeof(double) * rows * 4);
    for (int sweep = 0; sweep < 60; sweep++) {
        bool rotated = false;
        for (int p = 0; p < 3; p++)
            for (int q = p + 1; q < 4; q++) {
                double a = 0, b = 0, g = 0;
                for (int k = 0; k < rows; k++) {
                    a += U[4 * k + p] * U[4 * k + p];
                    b += U[4 * k + q] * U[4 * k + q];
                    g += U[4 * k + p] * U[4 * k + q];
                }
                if (g == 0 || std::fabs(g) <= 1e-17 * std::sqrt(a * b)) continue;
                rotated = true;
                const double zeta = (b - a) / (2 * g);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1 + zeta * zeta));
                const double c = 1 / std::sqrt(1 + t * t), s = c * t;
                for (int k = 0; k < rows; k++) {
                    const double up = U[4 * k + p], uq = U[4 * k + q];
                    U[4 * k + p] = c * up - s * uq;
                    U[4 * k + q] = s * up + c * uq;
                }
                for (int k = 0; k < 4; k++) {
                    const double vp = V[4 * k + p], vq = V[4 * k + q];
                    V[4 * k + p] = c * vp - s * vq;
                    V[4 * k + q] = s * vp + c * vq;
                }
            }
        if (!rotated) break;
    }
    int best = 0;
    double bn = 1e300;
    for (int j = 0; j < 4; j++) {
        double s = 0;
        for (int k = 0; k < rows; k++) s += U[4 * k + j] * U[4 * k + j];
        if (s < bn) bn = s, best = j;
    }
    for (int k = 0; k < 4; k++) v[k] = V[4 * k + best];
}

}  // namespace vb
