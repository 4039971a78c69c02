// Host implementation of the one-shot initialisation (see initial.h).  Own small dense linear algebra: the reference
// leans on Eigen / OpenCV / Ceres here, none of which is a dependency of this library.
#include "initial.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>

#include "fm_ransac.h"

namespace vb {
namespace init {

namespace {

inline double det3(const Mat3& a) {
    return a(0, 0) * (a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1)) - a(0, 1) * (a(1, 0) * a(2, 2) - a(1, 2) * a(2, 0)) +
           a(0, 2) * (a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0));
}
// qmul() with the y and z components summed in a different term order
inline Quat qmul_init(const Quat& a, const Quat& b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
inline Quat qconj(const Quat& a) { return {a.w, -a.x, -a.y, -a.z}; }
// q.R() * v, where qrot() is Eigen's quaternion * vector
inline Vec3 qrot_init(const Quat& q, const Vec3& v) { return q.R() * v; }

// rodrigues(), except that below |w| = 1e-12 it returns I + [w]x without the [w]x^2 / 2 term
Mat3 exp_so3(const Vec3& w) {
    if (w.norm() < 1e-12) return madd(Mat3(), skew(w));
    return rodrigues(w);
}

// Symmetric eigen-decomposition by cyclic Jacobi (n <= 4 here): A (n x n, destroyed) -> eigenvalues in d, vectors in V columns.
void jacobi_eig(double* A, int n, double* d, double* V) {
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) V[i * n + j] = i == j;
    for (int sweep = 0; sweep < 80; sweep++) {
        double off = 0;
        for (int p = 0; p < n; p++)
            for (int q = p + 1; q < n; q++) off += A[p * n + q] * A[p * n + q];
        if (off < 1e-300) break;
        for (int p = 0; p < n; p++)
            for (int q = p + 1; q < n; q++) {
                const double apq = A[p * n + q];
                if (apq == 0) continue;
                const double theta = (A[q * n + q] - A[p * n + p]) / (2 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
                const double c = 1 / std::sqrt(t * t + 1), s = t * c;
                for (int k = 0; k < n; k++) {
                    const double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s * akq;
                    A[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; k++) {
                    const double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s * aqk;
                    A[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; k++) {
                    const double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = c * vkp - s * vkq;
                    V[k * n + q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < n; i++) d[i] = A[i * n + i];
}

// SVD of a 3x3 matrix with det(U) = det(V) = +1 (the sign fix cv::decomposeEssentialMat applies afterwards).
void svd3_proper(const Mat3& E, Mat3& U, Mat3& V) {
    Mat3 EtE = E.T() * E;
    double d[3], Vv[9];
    jacobi_eig(EtE.m, 3, d, Vv);
    int o[3] = {0, 1, 2};
    std::sort(o, o + 3, [&](int a, int b) { return d[a] > d[b]; });
    Vec3 v[3], u[3];
    for (int k = 0; k < 2; k++) {
        v[k] = Vec3(Vv[0 * 3 + o[k]], Vv[1 * 3 + o[k]], Vv[2 * 3 + o[k]]);
        u[k] = E * v[k];
        u[k] = u[k] * (1.0 / u[k].norm());
    }
    // re-orthogonalise u1 against u0 (the two leading singular values of an essential matrix are close)
    u[1] = u[1] - u[0] * dot(u[0], u[1]);
    u[1] = u[1] * (1.0 / u[1].norm());
    v[2] = cross(v[0], v[1]);
    u[2] = cross(u[0], u[1]);
    for (int k = 0; k < 3; k++) {
        U(0, k) = u[k].x; U(1, k) = u[k].y; U(2, k) = u[k].z;
        V(0, k) = v[k].x; V(1, k) = v[k].y; V(2, k) = v[k].z;
    }
}

// Symmetric solve A x = b (A n x n row major, destroyed) by LDL^T with diagonal pivoting (Eigen's ldlt() scheme).
bool ldlt_solve(std::vector<double>& A, std::vector<double>& b, int n) {
    std::vector<int> perm(n);
    for (int i = 0; i < n; i++) perm[i] = i;
    for (int k = 0; k < n; k++) {
        int piv = k;
        double best = std::fabs(A[(size_t)k * n + k]);
        for (int i = k + 1; i < n; i++)
            if (std::fabs(A[(size_t)i * n + i]) > best) best = std::fabs(A[(size_t)i * n + i]), piv = i;
        if (best == 0 || !std::isfinite(best)) return false;
        if (piv != k) {
            for (int j = 0; j < n; j++) std::swap(A[(size_t)k * n + j], A[(size_t)piv * n + j]);
            for (int j = 0; j < n; j++) std::swap(A[(size_t)j * n + k], A[(size_t)j * n + piv]);
            std::swap(b[k], b[piv]);
            std::swap(perm[k], perm[piv]);
        }
        const double dkk = A[(size_t)k * n + k];
        for (int i = k + 1; i < n; i++) {
            const double lik = A[(size_t)i * n + k] / dkk;
            if (lik != 0)
                for (int j = k + 1; j < n; j++) A[(size_t)i * n + j] -= lik * A[(size_t)k * n + j];
            A[(size_t)i * n + k] = lik;
        }
    }
    for (int i = 0; i < n; i++)  // L y = P b
        for (int j = 0; j < i; j++) b[i] -= A[(size_t)i * n + j] * b[j];
    for (int i = 0; i < n; i++) b[i] /= A[(size_t)i * n + i];
    for (int i = n - 1; i >= 0; i--)  // L^T z = D^-1 y
        for (int j = i + 1; j < n; j++) b[i] -= A[(size_t)j * n + i] * b[j];
    std::vector<double> x(n);
    for (int i = 0; i < n; i++) x[perm[i]] = b[i];
    b.swap(x);
    return true;
}

// Cholesky solve of an SPD system (row major, destroyed); false when a pivot is not positive.
bool chol_solve(std::vector<double>& A, std::vector<double>& b, int n) {
    for (int j = 0; j < n; j++) {
        double d = A[j * n + j];
        for (int k = 0; k < j; k++) d -= A[j * n + k] * A[j * n + k];
        if (!(d > 0)) return false;
        d = std::sqrt(d);
        A[j * n + j] = d;
        for (int i = j + 1; i < n; i++) {
            double s = A[i * n + j];
            for (int k = 0; k < j; k++) s -= A[i * n + k] * A[j * n + k];
            A[i * n + j] = s / d;
        }
    }
    for (int i = 0; i < n; i++) {
        double s = b[i];
        for (int k = 0; k < i; k++) s -= A[i * n + k] * b[k];
        b[i] = s / A[i * n + i];
    }
    for (int i = n - 1; i >= 0; i--) {
        double s = b[i];
        for (int k = i + 1; k < n; k++) s -= A[k * n + i] * b[k];
        b[i] = s / A[i * n + i];
    }
    return true;
}

bool inv3_sym(const double* a, double* inv) {  // symmetric 3x3 (row major 9) inverse
    const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
    const double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
    if (det == 0 || !std::isfinite(det)) return false;
    const double id = 1.0 / det;
    inv[0] = c00 * id; inv[1] = (a[2] * a[7] - a[1] * a[8]) * id; inv[2] = (a[1] * a[5] - a[2] * a[4]) * id;
    inv[3] = c01 * id; inv[4] = (a[0] * a[8] - a[2] * a[6]) * id; inv[5] = (a[2] * a[3] - a[0] * a[5]) * id;
    inv[6] = c02 * id; inv[7] = (a[1] * a[6] - a[0] * a[7]) * id; inv[8] = (a[0] * a[4] - a[1] * a[3]) * id;
    return true;
}

void pose34(const Mat3& R, const Vec3& t, double P[12]) {
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) P[4 * i + j] = R(i, j);
        P[4 * i + 3] = t[i];
    }
}

}  // namespace

// ---- Preint (factor/integration_base.h:33-186) ----------------------------------------------------------------------------
void Preint::start(const Vec3& a0, const Vec3& g0, const Vec3& ba_, const Vec3& bg_) {
    lin_acc = acc_0 = a0;
    lin_gyr = gyr_0 = g0;
    ba = ba_;
    bg = bg_;
    dt.clear(); acc.clear(); gyr.clear();
    sum_dt = 0;
    dp = dv = Vec3();
    dq = Quat();
    J_R_bg = mscale(Mat3(), 0.0);
    valid = true;
}
void Preint::propagate(double dt_, const Vec3& a1, const Vec3& g1) {
    const Vec3 un_acc_0 = qrot_init(dq, acc_0 - ba);
    const Vec3 un_gyr = 0.5 * (gyr_0 + g1) - bg;
    Quat rq = qmul_init(dq, Quat(1, un_gyr.x * dt_ / 2, un_gyr.y * dt_ / 2, un_gyr.z * dt_ / 2));
    const Vec3 un_acc_1 = qrot_init(rq, a1 - ba);
    const Vec3 un_acc = 0.5 * (un_acc_0 + un_acc_1);
    dp = dp + dv * dt_ + 0.5 * un_acc * dt_ * dt_;
    dv = dv + un_acc * dt_;
    // jacobian = F * jacobian, rows O_R: F(3,3) = I - [w]x dt, F(3,12) = -I dt (integration_base.h:104-105)
    J_R_bg = madd(madd(Mat3(), mscale(skew(un_gyr), -dt_)) * J_R_bg, mscale(Mat3(), -dt_));
    dq = rq.normalized();
    sum_dt += dt_;
    acc_0 = a1;
    gyr_0 = g1;
}
void Preint::push_back(double dt_, const Vec3& a, const Vec3& g) {
    dt.push_back(dt_);
    acc.push_back(a);
    gyr.push_back(g);
    propagate(dt_, a, g);
}
void Preint::repropagate(const Vec3& ba_, const Vec3& bg_) {
    sum_dt = 0;
    acc_0 = lin_acc;
    gyr_0 = lin_gyr;
    dp = dv = Vec3();
    dq = Quat();
    ba = ba_;
    bg = bg_;
    J_R_bg = mscale(Mat3(), 0.0);
    for (size_t i = 0; i < dt.size(); i++) propagate(dt[i], acc[i], gyr[i]);
}

// ---- two-view geometry -----------------------------------------------------------------------------------------------------
Vec3 triangulate_point(const double P0[12], const double P1[12], const double x0[2], const double x1[2]) {
    double A[16], v[4];
    for (int c = 0; c < 4; c++) {
        A[0 + c] = x0[0] * P0[8 + c] - P0[0 + c];
        A[4 + c] = x0[1] * P0[8 + c] - P0[4 + c];
        A[8 + c] = x1[0] * P1[8 + c] - P1[0 + c];
        A[12 + c] = x1[1] * P1[8 + c] - P1[4 + c];
    }
    null_direction4(A, 4, v);
    return Vec3(v[0] / v[3], v[1] / v[3], v[2] / v[3]);
}

int recover_pose(const double E[9], const float* p1, const float* p2, int n, unsigned char* mask, Mat3& R, Vec3& t) {
    Mat3 Em, U, V;
    std::memcpy(Em.m, E, sizeof(Em.m));
    svd3_proper(Em, U, V);
    Mat3 W = mscale(Mat3(), 0.0);
    W(0, 1) = 1; W(1, 0) = -1; W(2, 2) = 1;
    const Mat3 R1 = U * W * V.T(), R2 = U * W.T() * V.T();
    const Vec3 t0 = U.col(2);
    const Mat3 Rs[4] = {R1, R2, R1, R2};
    const Vec3 ts[4] = {t0, t0, t0 * -1.0, t0 * -1.0};
    const double dist = 50.0;
    double P0[12];
    pose34(Mat3(), Vec3(), P0);
    std::vector<unsigned char> m[4];
    int good[4];
    for (int c = 0; c < 4; c++) {
        double P[12];
        pose34(Rs[c], ts[c], P);
        m[c].assign(n, 0);
        good[c] = 0;
        for (int i = 0; i < n; i++) {
            const double x0[2] = {(double)p1[2 * i], (double)p1[2 * i + 1]}, x1[2] = {(double)p2[2 * i], (double)p2[2 * i + 1]};
            double A[16], q[4];
            for (int k = 0; k < 4; k++) {
                A[0 + k] = x0[0] * P0[8 + k] - P0[0 + k];
                A[4 + k] = x0[1] * P0[8 + k] - P0[4 + k];
                A[8 + k] = x1[0] * P[8 + k] - P[0 + k];
                A[12 + k] = x1[1] * P[8 + k] - P[4 + k];
            }
            null_direction4(A, 4, q);
            bool ok = q[2] * q[3] > 0;
            const Vec3 X(q[0] / q[3], q[1] / q[3], q[2] / q[3]);
            ok = ok && X.z < dist;
            const double z2 = P[8] * X.x + P[9] * X.y + P[10] * X.z + P[11];
            ok = ok && z2 > 0 && z2 < dist;
            if (mask) ok = ok && mask[i];
            m[c][i] = ok;
            good[c] += ok;
        }
    }
    int pick;
    if (good[0] >= good[1] && good[0] >= good[2] && good[0] >= good[3]) pick = 0;
    else if (good[1] >= good[0] && good[1] >= good[2] && good[1] >= good[3]) pick = 1;
    else if (good[2] >= good[0] && good[2] >= good[1] && good[2] >= good[3]) pick = 2;
    else pick = 3;
    R = Rs[pick];
    t = ts[pick];
    if (mask) std::memcpy(mask, m[pick].data(), n);
    return good[pick];
}

bool solve_relative_rt(const std::vector<double>& corres4, Mat3& Rotation, Vec3& Translation, int* inliers) {
    const int n = (int)(corres4.size() / 4);
    if (inliers) *inliers = 0;
    if (n < 15) return false;
    std::vector<float> ll(2 * n), rr(2 * n);
    for (int i = 0; i < n; i++) {
        ll[2 * i] = (float)corres4[4 * i]; ll[2 * i + 1] = (float)corres4[4 * i + 1];
        rr[2 * i] = (float)corres4[4 * i + 2]; rr[2 * i + 1] = (float)corres4[4 * i + 3];
    }
    std::vector<unsigned char> mask(n);
    double E[9];
    if (!vb::fundamental_ransac(ll.data(), rr.data(), n, 0.3 / 460, 0.99, mask.data(), E)) return false;
    Mat3 R;
    Vec3 T;
    const int cnt = recover_pose(E, ll.data(), rr.data(), n, mask.data(), R, T);
    Rotation = R.T();
    Translation = (R.T() * T) * -1.0;
    if (inliers) *inliers = cnt;
    return cnt > 12;
}

// ---- solvePnP (iterative, from a guess) ------------------------------------------------------------------------------------
bool solve_pnp(const std::vector<double>& pts3, const std::vector<double>& pts2, Mat3& R, Vec3& t) {
    const int n = (int)(pts2.size() / 2);
    if (n < 4) return false;
    std::vector<Vec3> X(n);
    std::vector<double> u(n), v(n);
    for (int i = 0; i < n; i++) {  // cv::Point3f / cv::Point2f
        X[i] = Vec3((float)pts3[3 * i], (float)pts3[3 * i + 1], (float)pts3[3 * i + 2]);
        u[i] = (float)pts2[2 * i];
        v[i] = (float)pts2[2 * i + 1];
    }
    auto cost_of = [&](const Mat3& Rm, const Vec3& tv) {
        double c = 0;
        for (int i = 0; i < n; i++) {
            const Vec3 p = Rm * X[i] + tv;
            const double ex = p.x / p.z - u[i], ey = p.y / p.z - v[i];
            c += ex * ex + ey * ey;
        }
        return c;
    };
    double lambda = 1e-3, cost = cost_of(R, t);
    if (!std::isfinite(cost)) return false;
    for (int iter = 0; iter < 100; iter++) {
        double H[36] = {0}, g[6] = {0};
        for (int i = 0; i < n; i++) {
            const Vec3 RX = R * X[i], p = RX + t;
            const double iz = 1.0 / p.z, x = p.x * iz, y = p.y * iz;
            const double ex = x - u[i], ey = y - v[i];
            // d(x,y)/dp
            const double a[2][3] = {{iz, 0, -x * iz}, {0, iz, -y * iz}};
            // dp/dw = -[RX]x , dp/dt = I
            const Mat3 S = skew(RX);
            double J[2][6];
            for (int r = 0; r < 2; r++) {
                for (int c = 0; c < 3; c++) J[r][c] = -(a[r][0] * S(0, c) + a[r][1] * S(1, c) + a[r][2] * S(2, c));
                for (int c = 0; c < 3; c++) J[r][3 + c] = a[r][c];
            }
            for (int r = 0; r < 6; r++) {
                g[r] += J[0][r] * ex + J[1][r] * ey;
                for (int c = 0; c < 6; c++) H[6 * r + c] += J[0][r] * J[0][c] + J[1][r] * J[1][c];
            }
        }
        bool improved = false;
        double step_norm = 0;
        for (int attempt = 0; attempt < 30 && !improved; attempt++) {
            std::vector<double> A(H, H + 36), b(6);
            for (int k = 0; k < 6; k++) {
                A[7 * k] += lambda * (H[7 * k] > 0 ? H[7 * k] : 1.0);
                b[k] = -g[k];
            }
            if (!chol_solve(A, b, 6)) {
                lambda *= 10;
                continue;
            }
            const Mat3 Rn = exp_so3(Vec3(b[0], b[1], b[2])) * R;
            const Vec3 tn = t + Vec3(b[3], b[4], b[5]);
            const double cn = cost_of(Rn, tn);
            step_norm = std::sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2] + b[3] * b[3] + b[4] * b[4] + b[5] * b[5]);
            if (std::isfinite(cn) && cn <= cost) {
                R = Rn;
                t = tn;
                improved = true;
                const double drop = cost - cn;
                cost = cn;
                lambda = std::max(lambda * 0.1, 1e-12);
                if (drop <= 1e-16 * (cost + 1e-300)) step_norm = 0;  // flat: stop below
            } else
                lambda *= 10;
        }
        if (!improved || step_norm < 1e-13) break;
    }
    // keep R a rotation after the accumulated updates
    R = Quat::FromR(R).normalized().R();
    return true;
}

// ---- GlobalSFM (initial/initial_sfm.cpp) -----------------------------------------------------------------------------------
namespace {

struct SfmFeature {
    bool state = false;
    int id = 0;
    std::vector<std::pair<int, std::pair<double, double>>> obs;
    Vec3 pos;
};

bool solve_frame_by_pnp(Mat3& R_initial, Vec3& P_initial, int i, const std::vector<SfmFeature>& f) {
    std::vector<double> p2, p3;
    for (auto& ft : f) {
        if (!ft.state) continue;
        for (auto& o : ft.obs)
            if (o.first == i) {
                p2.push_back(o.second.first); p2.push_back(o.second.second);
                p3.push_back(ft.pos.x); p3.push_back(ft.pos.y); p3.push_back(ft.pos.z);
                break;
            }
    }
    if ((int)(p2.size() / 2) < 15) {
        if ((int)(p2.size() / 2) < 10) return false;
    }
    return solve_pnp(p3, p2, R_initial, P_initial);
}

void triangulate_two_frames(int frame0, const double* Pose0, int frame1, const double* Pose1, std::vector<SfmFeature>& f) {
    for (auto& ft : f) {
        if (ft.state) continue;
        bool has0 = false, has1 = false;
        double x0[2], x1[2];
        for (auto& o : ft.obs) {
            if (o.first == frame0) { x0[0] = o.second.first; x0[1] = o.second.second; has0 = true; }
            if (o.first == frame1) { x1[0] = o.second.first; x1[1] = o.second.second; has1 = true; }
        }
        if (has0 && has1) {
            ft.pos = triangulate_point(Pose0, Pose1, x0, x1);
            ft.state = true;
        }
    }
}

// The vision-only bundle of construct(): Ceres' trust-region Levenberg-Marquardt with DENSE_SCHUR and its default
// options (Ceres 1.14 TrustRegionMinimizer / LevenbergMarquardtStrategy: Jacobi scaling, radius 1e4, the
// 1 - (2 rho - 1)^3 radius rule, function / parameter / gradient tolerances 1e-6 / 1e-8 / 1e-10, 50 iterations).
// max_solver_time_in_seconds = 0.2 is a wall-clock cap and is not reproduced (machine dependent).
// Rotations are updated on the left, R <- exp(w) R, which is Ceres' QuaternionParameterization up to the factor 2 that
// the Jacobi scaling removes.  Returns true for CONVERGENCE.
bool sfm_bundle(int frame_num, int l, std::vector<Mat3>& cR, std::vector<Vec3>& cT, std::vector<SfmFeature>& f, int* iterations,
                double* final_cost, double function_tolerance) {
    struct Obs { int cam, pt; double u, v; };
    std::vector<int> pts;  // feature index per point block
    std::vector<Obs> obs;
    for (int i = 0; i < (int)f.size(); i++) {
        if (!f[i].state) continue;
        const int p = (int)pts.size();
        pts.push_back(i);
        for (auto& o : f[i].obs) obs.push_back({o.first, p, o.second.first, o.second.second});
    }
    const int np = (int)pts.size(), no = (int)obs.size();
    // camera parameter columns: rotation (3) unless i == l, translation (3) unless i == l or the last frame
    std::vector<int> rot_col(frame_num, -1), tr_col(frame_num, -1);
    int nc = 0;
    for (int i = 0; i < frame_num; i++) {
        if (i != l) { rot_col[i] = nc; nc += 3; }
        if (i != l && i != frame_num - 1) { tr_col[i] = nc; nc += 3; }
    }
    const int nx = nc + 3 * np;
    std::vector<Vec3> X(np);
    for (int p = 0; p < np; p++) X[p] = f[pts[p]].pos;

    auto residuals = [&](const std::vector<Mat3>& Rm, const std::vector<Vec3>& Tv, const std::vector<Vec3>& Xp, std::vector<double>& r) {
        r.resize(2 * no);
        double c = 0;
        for (int k = 0; k < no; k++) {
            const Vec3 p = Rm[obs[k].cam] * Xp[obs[k].pt] + Tv[obs[k].cam];
            r[2 * k] = p.x / p.z - obs[k].u;
            r[2 * k + 1] = p.y / p.z - obs[k].v;
            c += r[2 * k] * r[2 * k] + r[2 * k + 1] * r[2 * k + 1];
        }
        return 0.5 * c;
    };
    std::vector<double> r, Jc(12 * no), Jp(6 * no), scale(nx), gvec(nx), Hcc, Hpp;
    std::vector<std::vector<int>> by_pt(np);  // observations grouped by point (for the Schur complement)
    for (int k = 0; k < no; k++) by_pt[obs[k].pt].push_back(k);
    auto col_of = [&](int k, int c) {  // global column of camera-local column c of observation k (-1: constant block)
        return c < 3 ? (rot_col[obs[k].cam] < 0 ? -1 : rot_col[obs[k].cam] + c)
                     : (tr_col[obs[k].cam] < 0 ? -1 : tr_col[obs[k].cam] + c - 3);
    };
    double cost = residuals(cR, cT, X, r);
    double radius = 1e4, decrease_factor = 2.0;
    bool scale_set = false, converged = false, need_lin = true;
    int iter = 0;
    auto x_norm = [&]() {
        double s = 0;
        for (int i = 0; i < frame_num; i++) s += 1.0 + dot(cT[i], cT[i]);  // unit quaternion + translation
        for (int p = 0; p < np; p++) s += dot(X[p], X[p]);
        return std::sqrt(s);
    };
    auto linearise = [&]() {
        for (int k = 0; k < no; k++) {
            const Mat3& Rk = cR[obs[k].cam];
            const Vec3 RX = Rk * X[obs[k].pt], p = RX + cT[obs[k].cam];
            const double iz = 1.0 / p.z, x = p.x * iz, y = p.y * iz;
            const double a[2][3] = {{iz, 0, -x * iz}, {0, iz, -y * iz}};
            const Mat3 S = skew(RX);
            for (int rr = 0; rr < 2; rr++) {
                for (int c = 0; c < 3; c++) Jc[12 * k + 6 * rr + c] = -(a[rr][0] * S(0, c) + a[rr][1] * S(1, c) + a[rr][2] * S(2, c));
                for (int c = 0; c < 3; c++) Jc[12 * k + 6 * rr + 3 + c] = a[rr][c];
                for (int c = 0; c < 3; c++) Jp[6 * k + 3 * rr + c] = a[rr][0] * Rk(0, c) + a[rr][1] * Rk(1, c) + a[rr][2] * Rk(2, c);
            }
        }
        if (!scale_set) {  // Jacobi scaling, fixed at the first Jacobian: 1 / (1 + ||column||)
            std::fill(scale.begin(), scale.end(), 0.0);
            for (int k = 0; k < no; k++) {
                for (int c = 0; c < 6; c++) {
                    const int gc = col_of(k, c);
                    if (gc >= 0) scale[gc] += Jc[12 * k + c] * Jc[12 * k + c] + Jc[12 * k + 6 + c] * Jc[12 * k + 6 + c];
                }
                for (int c = 0; c < 3; c++) scale[nc + 3 * obs[k].pt + c] += Jp[6 * k + c] * Jp[6 * k + c] + Jp[6 * k + 3 + c] * Jp[6 * k + 3 + c];
            }
            for (auto& s : scale) s = 1.0 / (1.0 + std::sqrt(s));
            scale_set = true;
        }
        for (int k = 0; k < no; k++) {
            for (int c = 0; c < 6; c++) {
                const int gc = col_of(k, c);
                const double s = gc >= 0 ? scale[gc] : 0.0;
                Jc[12 * k + c] *= s;
                Jc[12 * k + 6 + c] *= s;
            }
            for (int c = 0; c < 3; c++) {
                const double s = scale[nc + 3 * obs[k].pt + c];
                Jp[6 * k + c] *= s;
                Jp[6 * k + 3 + c] *= s;
            }
        }
        // gradient and the block pieces of J^T J
        std::fill(gvec.begin(), gvec.end(), 0.0);
        Hcc.assign((size_t)nc * nc, 0.0);
        Hpp.assign(9 * (size_t)np, 0.0);
        for (int k = 0; k < no; k++) {
            const double r0 = r[2 * k], r1 = r[2 * k + 1];
            for (int c = 0; c < 6; c++) {
                const int gc = col_of(k, c);
                if (gc < 0) continue;
                gvec[gc] += Jc[12 * k + c] * r0 + Jc[12 * k + 6 + c] * r1;
                for (int d = 0; d < 6; d++) {
                    const int gd = col_of(k, d);
                    if (gd >= 0) Hcc[(size_t)gc * nc + gd] += Jc[12 * k + c] * Jc[12 * k + d] + Jc[12 * k + 6 + c] * Jc[12 * k + 6 + d];
                }
            }
            const int p = obs[k].pt;
            for (int c = 0; c < 3; c++) {
                gvec[nc + 3 * p + c] += Jp[6 * k + c] * r0 + Jp[6 * k + 3 + c] * r1;
                for (int d = 0; d < 3; d++) Hpp[9 * p + 3 * c + d] += Jp[6 * k + c] * Jp[6 * k + d] + Jp[6 * k + 3 + c] * Jp[6 * k + 3 + d];
            }
        }
    };
    if (!std::isfinite(cost) || no == 0 || nc == 0) {
        if (iterations) *iterations = 0;
        if (final_cost) *final_cost = cost;
        return false;
    }
    for (; iter < 50 && !converged; iter++) {
        if (need_lin) {
            linearise();
            need_lin = false;
            double gmax = 0;
            for (int i = 0; i < nx; i++) gmax = std::max(gmax, std::fabs(gvec[i] / scale[i]));  // unscaled gradient
            if (gmax <= 1e-10) { converged = true; break; }
        }
        // (J^T J + D^2) step = -g with D^2 = clamp(diag(J^T J), 1e-6, 1e32) / radius, points eliminated first
        std::vector<double> S(Hcc), rhs(nc), Vinv(9 * (size_t)np), dstep(nx);
        for (int i = 0; i < nc; i++) {
            S[(size_t)i * nc + i] += std::min(std::max(Hcc[(size_t)i * nc + i], 1e-6), 1e32) / radius;
            rhs[i] = -gvec[i];
        }
        bool ok = true;
        for (int p = 0; p < np && ok; p++) {
            double Vb[9];
            std::memcpy(Vb, &Hpp[9 * p], sizeof(Vb));
            for (int c = 0; c < 3; c++) Vb[4 * c] += std::min(std::max(Hpp[9 * p + 4 * c], 1e-6), 1e32) / radius;
            ok = inv3_sym(Vb, &Vinv[9 * p]);
            if (!ok) break;
            const double* Vi = &Vinv[9 * p];
            const double gp[3] = {-gvec[nc + 3 * p], -gvec[nc + 3 * p + 1], -gvec[nc + 3 * p + 2]};
            double Vg[3];
            for (int c = 0; c < 3; c++) Vg[c] = Vi[3 * c] * gp[0] + Vi[3 * c + 1] * gp[1] + Vi[3 * c + 2] * gp[2];
            const auto& ks = by_pt[p];
            std::vector<double> Wk(18 * ks.size()), WV(18 * ks.size());  // W_a = Jc_a^T Jp_a (6x3), W_a V^-1
            for (size_t a = 0; a < ks.size(); a++) {
                const int k = ks[a];
                for (int c = 0; c < 6; c++)
                    for (int d = 0; d < 3; d++)
                        Wk[18 * a + 3 * c + d] = Jc[12 * k + c] * Jp[6 * k + d] + Jc[12 * k + 6 + c] * Jp[6 * k + 3 + d];
                for (int c = 0; c < 6; c++)
                    for (int d = 0; d < 3; d++)
                        WV[18 * a + 3 * c + d] = Wk[18 * a + 3 * c] * Vi[d] + Wk[18 * a + 3 * c + 1] * Vi[3 + d] + Wk[18 * a + 3 * c + 2] * Vi[6 + d];
            }
            for (size_t a = 0; a < ks.size(); a++)
                for (int c = 0; c < 6; c++) {
                    const int gc = col_of(ks[a], c);
                    if (gc < 0) continue;
                    rhs[gc] -= Wk[18 * a + 3 * c] * Vg[0] + Wk[18 * a + 3 * c + 1] * Vg[1] + Wk[18 * a + 3 * c + 2] * Vg[2];
                    for (size_t b = 0; b < ks.size(); b++)
                        for (int d = 0; d < 6; d++) {
                            const int gd = col_of(ks[b], d);
                            if (gd < 0) continue;
                            S[(size_t)gc * nc + gd] -= WV[18 * a + 3 * c] * Wk[18 * b + 3 * d] + WV[18 * a + 3 * c + 1] * Wk[18 * b + 3 * d + 1] +
                                                       WV[18 * a + 3 * c + 2] * Wk[18 * b + 3 * d + 2];
                        }
                }
        }
        if (ok) ok = chol_solve(S, rhs, nc);
        double model_cost_change = 0;
        if (ok) {
            for (int i = 0; i < nc; i++) dstep[i] = rhs[i];
            for (int p = 0; p < np; p++) {
                double b3[3] = {-gvec[nc + 3 * p], -gvec[nc + 3 * p + 1], -gvec[nc + 3 * p + 2]};
                for (int k : by_pt[p])
                    for (int c = 0; c < 6; c++) {
                        const int gc = col_of(k, c);
                        if (gc < 0) continue;
                        for (int d = 0; d < 3; d++) b3[d] -= (Jc[12 * k + c] * Jp[6 * k + d] + Jc[12 * k + 6 + c] * Jp[6 * k + 3 + d]) * dstep[gc];
                    }
                const double* Vi = &Vinv[9 * p];
                for (int c = 0; c < 3; c++) dstep[nc + 3 * p + c] = Vi[3 * c] * b3[0] + Vi[3 * c + 1] * b3[1] + Vi[3 * c + 2] * b3[2];
            }
            for (int k = 0; k < no; k++) {  // model_cost_change = -(J d) . (r + J d / 2)
                double m0 = 0, m1 = 0;
                for (int c = 0; c < 6; c++) {
                    const int gc = col_of(k, c);
                    if (gc < 0) continue;
                    m0 += Jc[12 * k + c] * dstep[gc];
                    m1 += Jc[12 * k + 6 + c] * dstep[gc];
                }
                for (int c = 0; c < 3; c++) {
                    m0 += Jp[6 * k + c] * dstep[nc + 3 * obs[k].pt + c];
                    m1 += Jp[6 * k + 3 + c] * dstep[nc + 3 * obs[k].pt + c];
                }
                model_cost_change -= m0 * (r[2 * k] + 0.5 * m0) + m1 * (r[2 * k + 1] + 0.5 * m1);
            }
            ok = model_cost_change > 0 && std::isfinite(model_cost_change);
        }
        if (!ok) {  // invalid step: shrink the region like an unsuccessful one
            radius /= decrease_factor;
            decrease_factor *= 2;
            if (radius < 1e-32) break;
            continue;
        }
        double step_norm2 = 0;
        for (int i = 0; i < nx; i++) {
            dstep[i] *= scale[i];
            step_norm2 += dstep[i] * dstep[i];
        }
        std::vector<Mat3> nR(cR);
        std::vector<Vec3> nT(cT), nX(X);
        for (int i = 0; i < frame_num; i++) {
            if (rot_col[i] >= 0) nR[i] = exp_so3(Vec3(dstep[rot_col[i]], dstep[rot_col[i] + 1], dstep[rot_col[i] + 2])) * cR[i];
            if (tr_col[i] >= 0) nT[i] = cT[i] + Vec3(dstep[tr_col[i]], dstep[tr_col[i] + 1], dstep[tr_col[i] + 2]);
        }
        for (int p = 0; p < np; p++) nX[p] = X[p] + Vec3(dstep[nc + 3 * p], dstep[nc + 3 * p + 1], dstep[nc + 3 * p + 2]);
        std::vector<double> nr;
        const double ncost = residuals(nR, nT, nX, nr);
        if (std::sqrt(step_norm2) <= 1e-8 * (x_norm() + 1e-8)) {  // parameter tolerance
            converged = true;
            continue;
        }
        const double cost_change = cost - ncost;
        if (std::isfinite(ncost) && std::fabs(cost_change) <= function_tolerance * cost) {  // function tolerance
            if (cost_change > 0) { cR = nR; cT = nT; X = nX; cost = ncost; }
            converged = true;
            continue;
        }
        const double rho = cost_change / model_cost_change;
        if (std::isfinite(ncost) && rho > 1e-3) {
            cR = nR; cT = nT; X = nX; r = nr; cost = ncost;
            radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2 * rho - 1, 3)));
            decrease_factor = 2.0;
            need_lin = true;
        } else {
            radius /= decrease_factor;
            decrease_factor *= 2;
            if (radius < 1e-32) break;
        }
    }
    for (int i = 0; i < frame_num; i++) cR[i] = Quat::FromR(cR[i]).normalized().R();
    for (int p = 0; p < np; p++) f[pts[p]].pos = X[p];
    if (iterations) *iterations = iter;
    if (final_cost) *final_cost = cost;
    return converged;
}

}  // namespace

bool sfm_construct(int frame_num, std::vector<Quat>& q, std::vector<Vec3>& T, int l, const Mat3& relative_R, const Vec3& relative_T,
                   const std::vector<Track>& tracks, std::map<int, Vec3>& sfm_tracked_points, int* iterations, double* final_cost,
                   double function_tolerance) {
    std::vector<SfmFeature> f(tracks.size());
    for (size_t i = 0; i < tracks.size(); i++) {
        f[i].id = tracks[i].id;
        for (size_t k = 0; k < tracks[i].xy.size() / 2; k++)
            f[i].obs.push_back({tracks[i].start_frame + (int)k, {tracks[i].xy[2 * k], tracks[i].xy[2 * k + 1]}});
    }
    q.assign(frame_num, Quat());
    T.assign(frame_num, Vec3());
    q[frame_num - 1] = qmul_init(q[l], Quat::FromR(relative_R));
    T[frame_num - 1] = relative_T;
    std::vector<Mat3> cR(frame_num);
    std::vector<Vec3> cT(frame_num);
    std::vector<std::vector<double>> Pose(frame_num, std::vector<double>(12));
    auto set_pose = [&](int i) { pose34(cR[i], cT[i], Pose[i].data()); };
    cR[l] = qconj(q[l]).R();
    cT[l] = (cR[l] * T[l]) * -1.0;
    set_pose(l);
    cR[frame_num - 1] = qconj(q[frame_num - 1]).R();
    cT[frame_num - 1] = (cR[frame_num - 1] * T[frame_num - 1]) * -1.0;
    set_pose(frame_num - 1);
    for (int i = l; i < frame_num - 1; i++) {
        if (i > l) {
            Mat3 R_initial = cR[i - 1];
            Vec3 P_initial = cT[i - 1];
            if (!solve_frame_by_pnp(R_initial, P_initial, i, f)) return false;
            cR[i] = R_initial;
            cT[i] = P_initial;
            set_pose(i);
        }
        triangulate_two_frames(i, Pose[i].data(), frame_num - 1, Pose[frame_num - 1].data(), f);
    }
    for (int i = l + 1; i < frame_num - 1; i++) triangulate_two_frames(l, Pose[l].data(), i, Pose[i].data(), f);
    for (int i = l - 1; i >= 0; i--) {
        Mat3 R_initial = cR[i + 1];
        Vec3 P_initial = cT[i + 1];
        if (!solve_frame_by_pnp(R_initial, P_initial, i, f)) return false;
        cR[i] = R_initial;
        cT[i] = P_initial;
        set_pose(i);
        triangulate_two_frames(i, Pose[i].data(), l, Pose[l].data(), f);
    }
    for (auto& ft : f) {
        if (ft.state) continue;
        if (ft.obs.size() >= 2) {
            const double x0[2] = {ft.obs.front().second.first, ft.obs.front().second.second};
            const double x1[2] = {ft.obs.back().second.first, ft.obs.back().second.second};
            ft.pos = triangulate_point(Pose[ft.obs.front().first].data(), Pose[ft.obs.back().first].data(), x0, x1);
            ft.state = true;
        }
    }
    double cost = 0;
    const bool conv = sfm_bundle(frame_num, l, cR, cT, f, iterations, &cost, function_tolerance);
    if (final_cost) *final_cost = cost;
    if (!(conv || cost < 5e-03)) return false;
    for (int i = 0; i < frame_num; i++) {
        q[i] = qconj(Quat::FromR(cR[i]).normalized());
        T[i] = qrot_init(q[i], cT[i]) * -1.0;
    }
    for (auto& ft : f)
        if (ft.state) sfm_tracked_points[ft.id] = ft.pos;
    return true;
}

// ---- visual-inertial alignment (initial/initial_aligment.cpp) --------------------------------------------------------------
namespace {

void solve_gyroscope_bias(std::vector<ImageFrame>& fr, std::vector<Vec3>& Bgs, Vec3* delta_out) {
    double A[9] = {0}, b[3] = {0};
    for (size_t i = 0; i + 1 < fr.size(); i++) {
        const ImageFrame &fi = fr[i], &fj = fr[i + 1];
        const Quat q_ij = Quat::FromR(fi.R.T() * fj.R);
        const Mat3& J = fj.pre.J_R_bg;
        const Quat e = qmul_init(qconj(fj.pre.dq), q_ij);
        const Vec3 tb(2 * e.x, 2 * e.y, 2 * e.z);
        const Mat3 JtJ = J.T() * J;
        const Vec3 Jtb = J.T() * tb;
        for (int k = 0; k < 9; k++) A[k] += JtJ.m[k];
        b[0] += Jtb.x; b[1] += Jtb.y; b[2] += Jtb.z;
    }
    std::vector<double> Av(A, A + 9), bv(b, b + 3);
    Vec3 delta;
    if (ldlt_solve(Av, bv, 3)) delta = Vec3(bv[0], bv[1], bv[2]);
    if (delta_out) *delta_out = delta;
    for (auto& g : Bgs) g += delta;
    for (size_t i = 0; i + 1 < fr.size(); i++) fr[i + 1].pre.repropagate(Vec3(), Bgs[0]);
}

void tangent_basis(const Vec3& g0, Vec3& b, Vec3& c) {
    const Vec3 a = g0 * (1.0 / g0.norm());
    Vec3 tmp(0, 0, 1);
    if (a.x == tmp.x && a.y == tmp.y && a.z == tmp.z) tmp = Vec3(1, 0, 0);
    b = tmp - a * dot(a, tmp);
    b = b * (1.0 / b.norm());
    c = cross(a, b);
}

// Accumulates r_A = tmp_A^T tmp_A, r_b = tmp_A^T tmp_b of one frame pair into (A, b); tmp_A is 6 x (6 + tail).
void accumulate(std::vector<double>& A, std::vector<double>& b, int n_state, int i, int tail, const double* tmpA, const double* tmpb) {
    const int w = 6 + tail;
    std::vector<double> rA((size_t)w * w, 0.0), rb(w, 0.0);
    for (int r = 0; r < w; r++) {
        for (int c = 0; c < w; c++) {
            double s = 0;
            for (int k = 0; k < 6; k++) s += tmpA[k * w + r] * tmpA[k * w + c];
            rA[(size_t)r * w + c] = s;
        }
        double s = 0;
        for (int k = 0; k < 6; k++) s += tmpA[k * w + r] * tmpb[k];
        rb[r] = s;
    }
    auto G = [&](int r) { return r < 6 ? i * 3 + r : n_state - tail + (r - 6); };
    for (int r = 0; r < w; r++) {
        b[G(r)] += rb[r];
        for (int c = 0; c < w; c++) A[(size_t)G(r) * n_state + G(c)] += rA[(size_t)r * w + c];
    }
}

void refine_gravity(std::vector<ImageFrame>& fr, const Vec3& tic, double g_norm, Vec3& g, std::vector<double>& x) {
    Vec3 g0 = g * (g_norm / g.norm());
    const int n = (int)fr.size(), n_state = n * 3 + 2 + 1;
    for (int k = 0; k < 4; k++) {
        std::vector<double> A((size_t)n_state * n_state, 0.0), b(n_state, 0.0);
        Vec3 lx, ly;
        tangent_basis(g0, lx, ly);
        for (int i = 0; i + 1 < n; i++) {
            const ImageFrame &fi = fr[i], &fj = fr[i + 1];
            const double dt = fj.pre.sum_dt;
            const Mat3 RiT = fi.R.T(), Rij = RiT * fj.R;
            double tA[6 * 9] = {0}, tb[6];
            for (int d = 0; d < 3; d++) tA[d * 9 + d] = -dt;
            const Vec3 c6 = RiT * lx * (dt * dt / 2), c7 = RiT * ly * (dt * dt / 2), c8 = (RiT * (fj.T - fi.T)) * (1 / 100.0);
            const Vec3 p = fj.pre.dp + Rij * tic - tic - (RiT * g0) * (dt * dt / 2);
            for (int d = 0; d < 3; d++) {
                tA[d * 9 + 6] = c6[d]; tA[d * 9 + 7] = c7[d]; tA[d * 9 + 8] = c8[d];
                tb[d] = p[d];
            }
            const Vec3 d6 = RiT * lx * dt, d7 = RiT * ly * dt;
            const Vec3 v = fj.pre.dv - (RiT * g0) * dt;
            for (int d = 0; d < 3; d++) {
                tA[(3 + d) * 9 + d] = -1;
                for (int c = 0; c < 3; c++) tA[(3 + d) * 9 + 3 + c] = Rij(d, c);
                tA[(3 + d) * 9 + 6] = d6[d]; tA[(3 + d) * 9 + 7] = d7[d];
                tb[3 + d] = v[d];
            }
            accumulate(A, b, n_state, i, 3, tA, tb);
        }
        for (auto& a : A) a *= 1000.0;
        for (auto& a : b) a *= 1000.0;
        ldlt_solve(A, b, n_state);
        x = b;
        const double dg0 = x[n_state - 3], dg1 = x[n_state - 2];
        g0 = g0 + lx * dg0 + ly * dg1;
        g0 = g0 * (g_norm / g0.norm());
    }
    g = g0;
}

bool linear_alignment(std::vector<ImageFrame>& fr, const Vec3& tic, double g_norm, Vec3& g, std::vector<double>& x) {
    const int n = (int)fr.size(), n_state = n * 3 + 3 + 1;
    std::vector<double> A((size_t)n_state * n_state, 0.0), b(n_state, 0.0);
    for (int i = 0; i + 1 < n; i++) {
        const ImageFrame &fi = fr[i], &fj = fr[i + 1];
        const double dt = fj.pre.sum_dt;
        const Mat3 RiT = fi.R.T(), Rij = RiT * fj.R;
        double tA[6 * 10] = {0}, tb[6];
        const Vec3 c9 = (RiT * (fj.T - fi.T)) * (1 / 100.0);
        const Vec3 p = fj.pre.dp + Rij * tic - tic;
        for (int d = 0; d < 3; d++) {
            tA[d * 10 + d] = -dt;
            for (int c = 0; c < 3; c++) tA[d * 10 + 6 + c] = RiT(d, c) * dt * dt / 2;
            tA[d * 10 + 9] = c9[d];
            tb[d] = p[d];
            tA[(3 + d) * 10 + d] = -1;
            for (int c = 0; c < 3; c++) tA[(3 + d) * 10 + 3 + c] = Rij(d, c);
            for (int c = 0; c < 3; c++) tA[(3 + d) * 10 + 6 + c] = RiT(d, c) * dt;
            tb[3 + d] = fj.pre.dv[d];
        }
        accumulate(A, b, n_state, i, 4, tA, tb);
    }
    for (auto& a : A) a *= 1000.0;
    for (auto& a : b) a *= 1000.0;
    if (!ldlt_solve(A, b, n_state)) return false;
    x = b;
    double s = x[n_state - 1] / 100.0;
    g = Vec3(x[n_state - 4], x[n_state - 3], x[n_state - 2]);
    if (std::fabs(g.norm() - g_norm) > 1.0 || s < 0 || !std::isfinite(s)) return false;
    refine_gravity(fr, tic, g_norm, g, x);
    s = x.back() / 100.0;
    x.back() = s;
    return !(s < 0.0);
}

}  // namespace

bool visual_imu_alignment(std::vector<ImageFrame>& frames, std::vector<Vec3>& Bgs, const Vec3& tic, double g_norm, Vec3& g,
                          std::vector<double>& x, Vec3* delta_bg) {
    solve_gyroscope_bias(frames, Bgs, delta_bg);
    return linear_alignment(frames, tic, g_norm, g, x);
}

bool relative_pose(const std::vector<Track>& tracks, int W, Mat3& R, Vec3& T, int& l) {
    for (int i = 0; i < W; i++) {
        std::vector<double> corres;
        for (auto& it : tracks) {
            const int end = it.start_frame + (int)(it.xy.size() / 2) - 1;
            if (it.start_frame <= i && end >= W) {
                const int a = i - it.start_frame, b = W - it.start_frame;
                corres.push_back(it.xy[2 * a]); corres.push_back(it.xy[2 * a + 1]);
                corres.push_back(it.xy[2 * b]); corres.push_back(it.xy[2 * b + 1]);
            }
        }
        const int n = (int)(corres.size() / 4);
        if (n > 20) {
            double sum = 0;
            for (int j = 0; j < n; j++) sum += std::hypot(corres[4 * j] - corres[4 * j + 2], corres[4 * j + 1] - corres[4 * j + 3]);
            const double average_parallax = 1.0 * sum / n;
            if (average_parallax * 460 > 30 && solve_relative_rt(corres, R, T)) {
                l = i;
                return true;
            }
        }
    }
    return false;
}

Result initial_structure(std::vector<ImageFrame>& frames, const std::vector<double>& headers, const std::vector<Track>& tracks,
                         const Mat3& ric, const Vec3& tic, double g_norm, std::vector<Vec3>& Bgs, std::vector<double>& x,
                         double function_tolerance) {
    Result res;
    const int F = (int)headers.size();
    Mat3 relative_R;
    Vec3 relative_T;
    int l = -1;
    if (!relative_pose(tracks, F - 1, relative_R, relative_T, l)) {
        res.code = INIT_FAIL_RELATIVE_POSE;
        return res;
    }
    res.l = l;
    std::vector<Quat> Q;
    std::vector<Vec3> T;
    std::map<int, Vec3> pts;
    if (!sfm_construct(F, Q, T, l, relative_R, relative_T, tracks, pts, &res.sfm_iterations, &res.sfm_cost, function_tolerance)) {
        res.code = INIT_FAIL_SFM;
        return res;
    }
    // solve pnp for all frames (estimator.cpp:291-357)
    int i = 0;
    for (auto& fr : frames) {
        if (i >= F) {
            res.code = INIT_FAIL_PNP;
            return res;
        }
        if (fr.t == headers[i]) {
            fr.is_key_frame = true;
            fr.R = Q[i].R() * ric.T();
            fr.T = T[i];
            i++;
            continue;
        }
        if (fr.t > headers[i]) i++;
        Mat3 R_initial = qconj(Q[i]).R();
        Vec3 P_initial = (R_initial * T[i]) * -1.0;
        fr.is_key_frame = false;
        std::vector<double> p3, p2;
        for (size_t k = 0; k < fr.ids.size(); k++) {
            auto it = pts.find(fr.ids[k]);
            if (it == pts.end()) continue;
            p3.push_back(it->second.x); p3.push_back(it->second.y); p3.push_back(it->second.z);
            p2.push_back(fr.xy[2 * k]); p2.push_back(fr.xy[2 * k + 1]);
        }
        if (p2.size() / 2 < 6 || !solve_pnp(p3, p2, R_initial, P_initial)) {
            res.code = INIT_FAIL_PNP;
            return res;
        }
        const Mat3 R_pnp = R_initial.T();
        fr.R = R_pnp * ric.T();
        fr.T = (R_pnp * P_initial) * -1.0;
    }
    Vec3 g;
    if (!visual_imu_alignment(frames, Bgs, tic, g_norm, g, x, &res.delta_bg)) {
        res.code = INIT_FAIL_ALIGN;
        return res;
    }
    res.g = g;
    res.scale = x.back();
    for (size_t k = 0; k < frames.size(); k++) res.frame_vel.push_back(Vec3(x[3 * k], x[3 * k + 1], x[3 * k + 2]));
    return res;
}

Mat3 g2R(const Vec3& g) {
    const Vec3 a = g * (1.0 / g.norm()), b(0, 0, 1);
    // Eigen::Quaterniond::FromTwoVectors(a, b)
    Quat q;
    const double c = dot(a, b);
    if (c < -1 + 1e-12) {
        // antiparallel: any axis orthogonal to a (Eigen takes it from an SVD; the branch is unreachable for a gravity estimate
        // that passed the |g| check with z up)
        Vec3 axis = cross(a, Vec3(1, 0, 0));
        if (axis.norm() < 1e-6) axis = cross(a, Vec3(0, 1, 0));
        axis = axis * (1.0 / axis.norm());
        q = Quat(0, axis.x, axis.y, axis.z);
    } else {
        const Vec3 axis = cross(a, b);
        const double s = std::sqrt((1 + c) * 2);
        q = Quat(s * 0.5, axis.x / s, axis.y / s, axis.z / s);
    }
    Mat3 R0 = q.R();
    const double yaw = R2ypr(R0).x;
    return ypr2R(Vec3(-yaw, 0, 0)) * R0;
}

}  // namespace init
}  // namespace vb

// ---- InitialEXRotation (initial/initial_ex_rotation.cpp): camera-IMU rotation from paired camera / gyroscope rotations -------------
namespace vb {
namespace init {

namespace {

// testTriangulation (:100-126): fraction of the correspondences in front of both cameras [I | 0] and [R | t]; the projection
// matrices pass through float like the reference's cv::Matx34f.
double test_triangulation(const std::vector<float>& l, const std::vector<float>& r, const Mat3& R, const Vec3& t) {
    const int n = (int)(l.size() / 2);
    double P0[12], P1[12];
    pose34(Mat3(), Vec3(), P0);
    Mat3 Rf;
    for (int k = 0; k < 9; k++) Rf.m[k] = (double)(float)R.m[k];
    pose34(Rf, Vec3((double)(float)t.x, (double)(float)t.y, (double)(float)t.z), P1);
    int front = 0;
    for (int i = 0; i < n; i++) {
        const double x0[2] = {(double)l[2 * i], (double)l[2 * i + 1]}, x1[2] = {(double)r[2 * i], (double)r[2 * i + 1]};
        const Vec3 X = triangulate_point(P0, P1, x0, x1);  // already divided by the homogeneous coordinate
        const double zr = P1[8] * X.x + P1[9] * X.y + P1[10] * X.z + P1[11];
        if (X.z > 0 && zr > 0) front++;
    }
    return n ? 1.0 * front / n : 0.0;
}

}  // namespace

Mat3 ExRotation::solve_relative_r(const std::vector<double>& corres4) const {
    const int n = (int)(corres4.size() / 4);
    if (n < 9) return Mat3();
    std::vector<float> ll(2 * n), rr(2 * n);
    for (int i = 0; i < n; i++) {
        ll[2 * i] = (float)corres4[4 * i]; ll[2 * i + 1] = (float)corres4[4 * i + 1];
        rr[2 * i] = (float)corres4[4 * i + 2]; rr[2 * i + 1] = (float)corres4[4 * i + 3];
    }
    // cv::findFundamentalMat(ll, rr): FM_RANSAC with its default threshold 3 and confidence 0.99 (on normalised coordinates every
    // hypothesis explains every point, so the first 7-point sample wins: the reference's behaviour, reproduced with the same RNG)
    std::vector<unsigned char> mask(n);
    double E[9];
    if (!vb::fundamental_ransac(ll.data(), rr.data(), n, 3.0, 0.99, mask.data(), E)) return Mat3();
    Mat3 Em, U, V;
    std::memcpy(Em.m, E, sizeof(Em.m));
    svd3_proper(Em, U, V);  // det U = det V = +1: the rotations below are proper, which is what the reference's E = -E retry achieves
    Mat3 W = mscale(Mat3(), 0.0);
    W(0, 1) = -1; W(1, 0) = 1; W(2, 2) = 1;
    const Mat3 R1 = U * W * V.T(), R2 = U * W.T() * V.T();
    const Vec3 t1 = U.col(2), t2 = U.col(2) * -1.0;
    const double ratio1 = std::max(test_triangulation(ll, rr, R1, t1), test_triangulation(ll, rr, R1, t2));
    const double ratio2 = std::max(test_triangulation(ll, rr, R2, t1), test_triangulation(ll, rr, R2, t2));
    const Mat3 ans = ratio1 > ratio2 ? R1 : R2;
    return ans.T();  // ans_R_eigen(j, i) = ans_R_cv(i, j)
}

bool ExRotation::calibrate(const std::vector<double>& corres4, const Quat& delta_q_imu, int window_size, Mat3& calib_ric_result,
                           const Mat3* rc_given) {
    frame_count++;
    Rc.push_back(rc_given ? *rc_given : solve_relative_r(corres4));
    Rimu.push_back(delta_q_imu.R());
    Rc_g.push_back(ric.T() * delta_q_imu.R() * ric);
    double AtA[16] = {0};
    for (int i = 1; i <= frame_count; i++) {
        const Quat r1 = Quat::FromR(Rc[i]), r2 = Quat::FromR(Rc_g[i]);
        // Quaterniond::angularDistance: 2 atan2(|vec(d)|, |w(d)|) of d = r1 * r2^-1
        const Quat dq = qmul_init(r1, qconj(r2));
        const double angular_distance = 180 / M_PI * 2.0 * std::atan2(std::sqrt(dq.x * dq.x + dq.y * dq.y + dq.z * dq.z), std::fabs(dq.w));
        const double huber = angular_distance > 5.0 ? 5.0 / angular_distance : 1.0;
        double L[16], Rm[16];
        auto fill = [](double* M, const Quat& q, double sgn) {  // [w I + sgn [q]x, q; -q^T, w]
            const Mat3 S = skew(Vec3(q.x, q.y, q.z));
            for (int a = 0; a < 3; a++) {
                for (int b = 0; b < 3; b++) M[4 * a + b] = (a == b ? q.w : 0.0) + sgn * S(a, b);
                M[4 * a + 3] = a == 0 ? q.x : a == 1 ? q.y : q.z;
                M[12 + a] = -(a == 0 ? q.x : a == 1 ? q.y : q.z);
            }
            M[15] = q.w;
        };
        fill(L, r1, 1.0);
        fill(Rm, Quat::FromR(Rimu[i]), -1.0);
        double B[16];
        for (int k = 0; k < 16; k++) B[k] = huber * (L[k] - Rm[k]);
        for (int a = 0; a < 4; a++)
            for (int b = 0; b < 4; b++) {
                double s = 0;
                for (int k = 0; k < 4; k++) s += B[4 * k + a] * B[4 * k + b];
                AtA[4 * a + b] += s;
            }
    }
    double d[4], Vv[16];
    jacobi_eig(AtA, 4, d, Vv);
    int o[4] = {0, 1, 2, 3};
    std::sort(o, o + 4, [&](int a, int b) { return d[a] > d[b]; });
    const int s = o[3];  // smallest singular value: svd.matrixV().col(3), quaternion coefficients in (x, y, z, w) order
    const Quat est = Quat(Vv[12 + s], Vv[0 + s], Vv[4 + s], Vv[8 + s]).normalized();
    ric = est.R().T();
    const double ric_cov1 = std::sqrt(std::max(d[o[2]], 0.0));  // svd.singularValues().tail<3>()(1)
    last_cov1 = ric_cov1;
    if (frame_count >= window_size && ric_cov1 > 0.25) {
        calib_ric_result = ric;
        return true;
    }
    return false;
}

}  // namespace init
}  // namespace vb
