// CameraPtr::liftProjective followed by the division by z, for host and device code alike: the tracker lifts its points
// on the host (tracker.cu), loop verification lifts the key frames' FAST corners on the device (lv_kernels.cu).
//   PINHOLE         PinholeCamera.cc:450-510           intrinsics = fx fy cx cy k1 k2 p1 p2
//   MEI             CataCamera.cc:556-625              intrinsics = gamma1 gamma2 u0 v0 k1 k2 p1 p2, plus xi
//   KANNALA_BRANDT  EquidistantCamera.cc:428-442       intrinsics = mu mv u0 v0 k2 k3 k4 k5
// Both sides compile without FMA contraction (--fmad=false, -ffp-contract=off) and use IEEE division and sqrt, so PINHOLE
// and MEI give the same doubles on host and device; KANNALA_BRANDT finds the same theta on both, and only atan2, sin and
// cos may differ in their last bits.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define CAM_FN __host__ __device__ inline
#else
#define CAM_FN inline
#endif

namespace vb {

// the values of vt_camera_model and vp_camera_model
constexpr int CAM_PINHOLE = 0, CAM_MEI = 1, CAM_KANNALA_BRANDT = 2;

// Recursive inverse of the radial-tangential distortion, n = 8 (PinholeCamera.cc:487-503, CataCamera.cc:596-611).
CAM_FN void undistort_radtan(double k1, double k2, double p1, double p2, double mx_d, double my_d, double& ux, double& uy) {
    ux = mx_d;
    uy = my_d;
    for (int i = 0; i < 8; ++i) {
        const double x2 = ux * ux, y2 = uy * uy, xy = ux * uy, rho2 = x2 + y2;
        const double rad = k1 * rho2 + k2 * rho2 * rho2;
        const double ddx = ux * rad + 2.0 * p1 * xy + p2 * (rho2 + 2.0 * x2);
        const double ddy = uy * rad + 2.0 * p2 * xy + p1 * (rho2 + 2.0 * y2);
        ux = mx_d - ddx;
        uy = my_d - ddy;
    }
}

CAM_FN double kb_poly(const double k[4], double t, double r) {
    const double t2 = t * t;
    return t * (1.0 + t2 * (k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3])))) - r;
}

CAM_FN double kb_dpoly(const double k[4], double t) {
    const double t2 = t * t;
    return 1.0 + t2 * (3.0 * k[0] + t2 * (5.0 * k[1] + t2 * (7.0 * k[2] + t2 * 9.0 * k[3])));
}

// EquidistantCamera::backprojectSymmetric (EquidistantCamera.cc:716-818): the smallest non-negative real root of
// k5 t^9 + k4 t^7 + k3 t^5 + k2 t^3 + t - r = 0, r itself when there is none.  The reference takes it from the eigenvalues of
// the companion matrix; here the first sign change of the polynomial on a fine grid is bracketed and polished by
// bisection + Newton (the same root to rounding).
CAM_FN double kb_theta(const double kin[4], double r) {
    // the reference lowers the polynomial degree by 2 for EVERY zero coefficient, whichever it is, and drops the terms above
    // the resulting degree (EquidistantCamera.cc:733-770)
    int npow = 9;
    for (int i = 0; i < 4; i++) npow -= kin[i] == 0.0 ? 2 : 0;
    if (npow == 1) return r;
    double k[4];
    for (int i = 0; i < 4; i++) k[i] = 2 * i + 3 <= npow ? kin[i] : 0.0;
    if (r <= 1e-10) return 0.0;  // f(0) = -r: the root is within the reference's tolerance of zero
    const double step = 1.0 / 512.0;
    double lo = 0.0;
    for (int i = 1; i <= 4096; i++) {  // up to theta = 8 rad, far beyond any lens
        double hi = i * step;
        if (kb_poly(k, hi, r) >= 0.0) {
            for (int it = 0; it < 24; it++) {  // bisection narrows the bracket, Newton finishes
                const double mid = 0.5 * (lo + hi);
                if (kb_poly(k, mid, r) < 0.0) lo = mid; else hi = mid;
            }
            double t = 0.5 * (lo + hi);
            for (int it = 0; it < 20; it++) {
                const double d = kb_dpoly(k, t);
                if (d == 0.0) break;
                const double tn = t - kb_poly(k, t, r) / d;
                if (!(tn >= lo && tn <= hi)) break;
                if (tn == t) break;
                t = tn;
            }
            return t;
        }
        lo = hi;
    }
    return r;
}

// (px, py) -> (X, Y) = liftProjective / z for camera_model CAM_*, intrinsics c in the model's order above
CAM_FN void lift_projective(int camera_model, const double c[8], double xi, double px, double py, double& X, double& Y) {
    const double fx = c[0], fy = c[1], cx = c[2], cy = c[3], k1 = c[4], k2 = c[5], p1 = c[6], p2 = c[7];
    const double mx_d = (1.0 / fx) * px + (-cx / fx), my_d = (1.0 / fy) * py + (-cy / fy);
    if (camera_model == CAM_KANNALA_BRANDT) {
        const double r = sqrt(mx_d * mx_d + my_d * my_d);
        const double phi = r < 1e-10 ? 0.0 : atan2(my_d, mx_d);
        const double theta = kb_theta(&c[4], r);
        const double Px = sin(theta) * cos(phi), Py = sin(theta) * sin(phi), Pz = cos(theta);
        X = Px / Pz;
        Y = Py / Pz;
        return;
    }
    double ux = mx_d, uy = my_d;
    if (!(k1 == 0.0 && k2 == 0.0 && p1 == 0.0 && p2 == 0.0)) undistort_radtan(k1, k2, p1, p2, mx_d, my_d, ux, uy);
    if (camera_model == CAM_MEI) {
        double Pz;
        if (xi == 1.0)
            Pz = (1.0 - ux * ux - uy * uy) / 2.0;
        else {
            const double rho2 = ux * ux + uy * uy;
            Pz = 1.0 - xi * (rho2 + 1.0) / (xi + sqrt(1.0 + (1.0 - xi * xi) * rho2));
        }
        X = ux / Pz;
        Y = uy / Pz;
        return;
    }
    X = ux;
    Y = uy;
}

}  // namespace vb

#undef CAM_FN
