// Residual/Jacobian evaluation of the VINS factors on the device (float64); the rotation arithmetic is rotation.h's.
//   ProjectionFactor::Evaluate      vins_estimator/src/factor/projection_factor.cpp:21-121
//   ProjectionTdFactor::Evaluate    vins_estimator/src/factor/projection_td_factor.cpp:34-141
//   IMUFactor::Evaluate             vins_estimator/src/factor/imu_factor.h:19-179
//   IntegrationBase::evaluate       vins_estimator/src/factor/integration_base.h:160-186
//   PoseLocalParameterization::Plus vins_estimator/src/factor/pose_local_parameterization.cpp:3-18
//   Cauchy corrector                vins_estimator/src/factor/marginalization_factor.cpp:37-68
// Jacobians are produced directly in the 6-dof tangent parameterisation (the 7th column of the
// reference's 2x7 / 15x7 blocks is identically zero and ComputeJacobian is [I6; 0]).
#pragma once
#include "ba_types.h"
#include "rotation.h"

namespace vb {

__device__ __forceinline__ Quat q_from_param(const double* p) { return Quat{p[6], p[3], p[4], p[5]}; }

// PoseLocalParameterization::Plus
__device__ __forceinline__ void pose_plus(const double* x, const double* d, double* out) {
    out[0] = x[0] + d[0];
    out[1] = x[1] + d[1];
    out[2] = x[2] + d[2];
    const Quat q = qnormalized(qmul(q_from_param(x), deltaQ(Vec3(d[3], d[4], d[5]))));
    out[3] = q.x;
    out[4] = q.y;
    out[5] = q.z;
    out[6] = q.w;
}

// ceres::CauchyLoss(1.0) + Corrector: returns 0.5*rho(s) and rescales r (2) and the Jacobian rows.
struct Corrector {
    double sqrt_rho1, residual_scaling, alpha_sq_norm, half_rho0;
};
__device__ __forceinline__ Corrector cauchy_corrector(double sq_norm) {
    Corrector c;
    const double sum = 1.0 + sq_norm, inv = 1.0 / sum;
    const double rho0 = log(sum), rho1 = fmax(2.2250738585072014e-308, inv), rho2 = -(inv * inv);
    c.half_rho0 = 0.5 * rho0;
    c.sqrt_rho1 = sqrt(rho1);
    if (sq_norm == 0.0 || rho2 <= 0.0) {
        // rho2 < 0 for Cauchy: Ceres/VINS take this branch (alpha = 0), marginalization_factor.cpp:49-53
        c.residual_scaling = c.sqrt_rho1;
        c.alpha_sq_norm = 0.0;
    } else {
        const double D = 1.0 + 2.0 * sq_norm * rho2 / rho1;
        const double alpha = 1.0 - sqrt(D);
        c.residual_scaling = c.sqrt_rho1 / (1 - alpha);
        c.alpha_sq_norm = alpha / sq_norm;
    }
    return c;
}

// One visual residual block.  J = [Ji(2x6) | Jj(2x6) | Jex(2x6) | Jl(2x1) | Jtd(2x1)] = 2 x 20.
struct VisualEval {
    double r[2];
    double J[2][20];
    double half_rho;
};

// EX / TD select at compile time whether the Jacobians with respect to the camera extrinsic (columns 12..17) and the
// time offset (column 19) are produced (constant parameter blocks get no Jacobian: ceres hands jacobians[k] == NULL).
template <bool EX, bool TD>
__device__ __forceinline__ void eval_visual(const BaDims& d, const double* pose_i, const double* pose_j, const double* ex,
                                            double inv_dep_i, double td, double pix, double piy, double pjx, double pjy,
                                            double vix, double viy, double vjx, double vjy, double td_i, double td_j,
                                            double row_i, double row_j, bool want_jac, bool robust, VisualEval& e) {
    Vec3 pts_i = Vec3(pix, piy, 1.0), pts_j = Vec3(pjx, pjy, 1.0);
    if (d.est_td) {  // ProjectionTdFactor
        const double ci = td - td_i + d.tr_over_row * (row_i - d.half_row);
        const double cj = td - td_j + d.tr_over_row * (row_j - d.half_row);
        pts_i = pts_i - ci * Vec3(vix, viy, 0.0);
        pts_j = pts_j - cj * Vec3(vjx, vjy, 0.0);
    }
    const Vec3 Pi = Vec3(pose_i[0], pose_i[1], pose_i[2]), Pj = Vec3(pose_j[0], pose_j[1], pose_j[2]), tic = Vec3(ex[0], ex[1], ex[2]);
    const Quat Qi = q_from_param(pose_i), Qj = q_from_param(pose_j), qic = q_from_param(ex);
    const Vec3 pci = Vec3(pts_i.x / inv_dep_i, pts_i.y / inv_dep_i, pts_i.z / inv_dep_i);
    const Vec3 pts_imu_i = qrot(qic, pci) + tic;
    const Vec3 pts_w = qrot(Qi, pts_imu_i) + Pi;
    const Vec3 pts_imu_j = qrot(qinv(Qj), pts_w - Pj);
    const Vec3 pcj = qrot(qinv(qic), pts_imu_j - tic);
    const double dep_j = pcj.z;
    const double s = d.sqrt_info_vis;
    e.r[0] = s * (pcj.x / dep_j - pts_j.x);
    e.r[1] = s * (pcj.y / dep_j - pts_j.y);
    const double sq = e.r[0] * e.r[0] + e.r[1] * e.r[1];
    Corrector c{1.0, 1.0, 0.0, 0.5 * sq};
    if (robust) c = cauchy_corrector(sq);
    e.half_rho = c.half_rho0;
    if (want_jac) {
        const Mat3 Ri = qR(Qi), Rj = qR(Qj), ric = qR(qic);
        const Mat3 ricT = mT(ric), RjT = mT(Rj);
        double red[2][3];
        red[0][0] = s * (1. / dep_j); red[0][1] = 0; red[0][2] = s * (-pcj.x / (dep_j * dep_j));
        red[1][0] = 0; red[1][1] = s * (1. / dep_j); red[1][2] = s * (-pcj.y / (dep_j * dep_j));
        const Mat3 A = mmul(ricT, RjT);                       // d pcj / d Pi
        const Mat3 B = mmul(mmul(A, Ri), mscale(skew(pts_imu_i), -1.0));
        const Mat3 Cm = mscale(A, -1.0);                      // d pcj / d Pj
        const Mat3 Dm = mmul(ricT, skew(pts_imu_j));
        const Mat3 tmp_r = mmul(mmul(A, Ri), ric);
        Mat3 Eex, Fex;
        if (EX) {
            Eex = mmul(ricT, msub(mmul(RjT, Ri), Mat3()));
            const Vec3 inner = mv(RjT, mv(Ri, tic) + Pi - Pj) - tic;
            Fex = madd(madd(mscale(mmul(tmp_r, skew(pci)), -1.0), skew(mv(tmp_r, pci))), skew(mv(ricT, inner)));
        }
        const Vec3 dl = mv(tmp_r, pts_i) * (-1.0 / (inv_dep_i * inv_dep_i));
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
#pragma unroll
            for (int cc = 0; cc < 3; cc++) {
                e.J[rr][cc] = red[rr][0] * A.m[cc] + red[rr][1] * A.m[3 + cc] + red[rr][2] * A.m[6 + cc];
                e.J[rr][3 + cc] = red[rr][0] * B.m[cc] + red[rr][1] * B.m[3 + cc] + red[rr][2] * B.m[6 + cc];
                e.J[rr][6 + cc] = red[rr][0] * Cm.m[cc] + red[rr][1] * Cm.m[3 + cc] + red[rr][2] * Cm.m[6 + cc];
                e.J[rr][9 + cc] = red[rr][0] * Dm.m[cc] + red[rr][1] * Dm.m[3 + cc] + red[rr][2] * Dm.m[6 + cc];
                if (EX) {
                    e.J[rr][12 + cc] = red[rr][0] * Eex.m[cc] + red[rr][1] * Eex.m[3 + cc] + red[rr][2] * Eex.m[6 + cc];
                    e.J[rr][15 + cc] = red[rr][0] * Fex.m[cc] + red[rr][1] * Fex.m[3 + cc] + red[rr][2] * Fex.m[6 + cc];
                } else {
                    e.J[rr][12 + cc] = 0.0;
                    e.J[rr][15 + cc] = 0.0;
                }
            }
            e.J[rr][18] = red[rr][0] * dl.x + red[rr][1] * dl.y + red[rr][2] * dl.z;
            e.J[rr][19] = 0.0;
        }
        if (TD && d.est_td) {
            const Vec3 vi = Vec3(vix, viy, 0.0);
            const Vec3 dtd = mv(tmp_r, vi) * (-1.0 / inv_dep_i);
            e.J[0][19] = red[0][0] * dtd.x + red[0][1] * dtd.y + red[0][2] * dtd.z + s * vjx;
            e.J[1][19] = red[1][0] * dtd.x + red[1][1] * dtd.y + red[1][2] * dtd.z + s * vjy;
        }
        if (robust) {
#pragma unroll
            for (int k = 0; k < 20; k++) {
                const double rtJ = e.r[0] * e.J[0][k] + e.r[1] * e.J[1][k];
                e.J[0][k] = c.sqrt_rho1 * (e.J[0][k] - c.alpha_sq_norm * e.r[0] * rtJ);
                e.J[1][k] = c.sqrt_rho1 * (e.J[1][k] - c.alpha_sq_norm * e.r[1] * rtJ);
            }
        }
    }
    if (robust) {
        e.r[0] *= c.residual_scaling;
        e.r[1] *= c.residual_scaling;
    }
}

// bottom-right 3x3 of Qleft(a) and of Qleft(a) * Qright(b)  (utility.h:51-68)
__device__ __forceinline__ Mat3 qleft_br(Quat q) { return madd(mscale(Mat3(), q.w), skew(Vec3(q.x, q.y, q.z))); }
__device__ __forceinline__ Mat3 qleft_qright_br(Quat a, Quat b) {
    // rows 1..3 of Qleft(a) times columns 1..3 of Qright(b)
    const Vec3 av = Vec3(a.x, a.y, a.z), bv = Vec3(b.x, b.y, b.z);
    const Mat3 La = madd(mscale(Mat3(), a.w), skew(av));
    const Mat3 Rb = msub(mscale(Mat3(), b.w), skew(bv));
    Mat3 r = mmul(La, Rb);
    // + a.vec * (-b.vec)^T  (column 0 of Qleft rows 1..3 times row 0 of Qright cols 1..3)
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) r.m[3 * i + j] += av[i] * (-bv[j]);
    return r;
}

// IMU factor: un-whitened residual (15) and Jacobian blocks written into Jraw[15][30] =
// [pose_i(6) | speedbias_i(9) | pose_j(6) | speedbias_j(9)] (row-major, zero-initialised by the caller).
__device__ inline void eval_imu_raw(const BaDims& d, const PreInt& pre, const double* pose_i, const double* sb_i,
                                    const double* pose_j, const double* sb_j, double* r, double* Jraw /* may be null */) {
    const Vec3 Pi = Vec3(pose_i[0], pose_i[1], pose_i[2]), Pj = Vec3(pose_j[0], pose_j[1], pose_j[2]);
    const Quat Qi = q_from_param(pose_i), Qj = q_from_param(pose_j);
    const Vec3 Vi = Vec3(sb_i[0], sb_i[1], sb_i[2]), Bai = Vec3(sb_i[3], sb_i[4], sb_i[5]), Bgi = Vec3(sb_i[6], sb_i[7], sb_i[8]);
    const Vec3 Vj = Vec3(sb_j[0], sb_j[1], sb_j[2]), Baj = Vec3(sb_j[3], sb_j[4], sb_j[5]), Bgj = Vec3(sb_j[6], sb_j[7], sb_j[8]);
    const Vec3 G = Vec3(d.G[0], d.G[1], d.G[2]);
    const double sum_dt = pre.sum_dt;
    auto blk = [&](int r0, int c0) {
        Mat3 b;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) b.m[3 * i + j] = pre.jac[(r0 + i) * 15 + c0 + j];
        return b;
    };
    const Mat3 dp_dba = blk(0, 9), dp_dbg = blk(0, 12), dq_dbg = blk(3, 12), dv_dba = blk(6, 9), dv_dbg = blk(6, 12);
    const Vec3 dba = Bai - Vec3(pre.ba[0], pre.ba[1], pre.ba[2]), dbg = Bgi - Vec3(pre.bg[0], pre.bg[1], pre.bg[2]);
    const Quat delta_q = Quat{pre.dq[0], pre.dq[1], pre.dq[2], pre.dq[3]};
    const Quat corrected_delta_q = qmul(delta_q, deltaQ(mv(dq_dbg, dbg)));
    const Vec3 corrected_delta_v = Vec3(pre.dv[0], pre.dv[1], pre.dv[2]) + mv(dv_dba, dba) + mv(dv_dbg, dbg);
    const Vec3 corrected_delta_p = Vec3(pre.dp[0], pre.dp[1], pre.dp[2]) + mv(dp_dba, dba) + mv(dp_dbg, dbg);
    const Quat Qi_inv = qinv(Qi);
    const Vec3 tp = qrot(Qi_inv, 0.5 * G * sum_dt * sum_dt + Pj - Pi - Vi * sum_dt);
    const Vec3 tv = qrot(Qi_inv, G * sum_dt + Vj - Vi);
    const Vec3 rp = tp - corrected_delta_p;
    const Quat qe = qmul(qinv(corrected_delta_q), qmul(Qi_inv, Qj));
    const Vec3 rq = 2.0 * Vec3(qe.x, qe.y, qe.z);
    const Vec3 rv = tv - corrected_delta_v;
    const Vec3 rba = Baj - Bai, rbg = Bgj - Bgi;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        r[i] = rp[i];
        r[3 + i] = rq[i];
        r[6 + i] = rv[i];
        r[9 + i] = rba[i];
        r[12 + i] = rbg[i];
    }
    if (!Jraw) return;
    auto put = [&](int r0, int c0, const Mat3& b) {
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) Jraw[(r0 + i) * 30 + c0 + j] = b.m[3 * i + j];
    };
    const Mat3 RiT = qR(Qi_inv), I3 = Mat3();
    // pose_i: cols 0..5
    put(0, 0, mscale(RiT, -1.0));
    put(0, 3, skew(tp));
    put(3, 3, mscale(qleft_qright_br(qmul(qinv(Qj), Qi), corrected_delta_q), -1.0));
    put(6, 3, skew(tv));
    // speedbias_i: cols 6..14 (v, ba, bg)
    put(0, 6, mscale(RiT, -sum_dt));
    put(0, 9, mscale(dp_dba, -1.0));
    put(0, 12, mscale(dp_dbg, -1.0));
    put(3, 12, mscale(mmul(qleft_br(qmul(qmul(qinv(Qj), Qi), delta_q)), dq_dbg), -1.0));
    put(6, 6, mscale(RiT, -1.0));
    put(6, 9, mscale(dv_dba, -1.0));
    put(6, 12, mscale(dv_dbg, -1.0));
    put(9, 9, mscale(I3, -1.0));
    put(12, 12, mscale(I3, -1.0));
    // pose_j: cols 15..20
    put(0, 15, RiT);
    put(3, 18, qleft_br(qmul(qmul(qinv(corrected_delta_q), Qi_inv), Qj)));
    // speedbias_j: cols 21..29
    put(6, 21, RiT);
    put(9, 24, I3);
    put(12, 27, I3);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace vb
