// One-shot visual-inertial initialisation on the host (SURVEY §8 next-1): what Estimator::initialStructure()
// (vins_estimator/src/estimator.cpp:218-471) computes from the first full window, stated on plain arrays so that the
// estimator shim and the handle-free ve_debug_init_* entries run the same code.
//   relative pose         initial/solve_5pts.cpp:193-227 (cv::findFundamentalMat + cv::recoverPose)
//   GlobalSFM::construct   initial/initial_sfm.cpp:117-312 (cv::solvePnP, SVD triangulation, Ceres bundle)
//   VisualIMUAlignment     initial/initial_aligment.cpp:3-207
// The reference runs this on the CPU as well (once per start or reboot); nothing here is a device hot path.
#pragma once
#include <map>
#include <vector>

#include "rotation.h"

namespace vb {
namespace init {


// The part of IntegrationBase (factor/integration_base.h:54-186) the initialiser reads: mid-point deltas, sum_dt and
// d(delta_q)/d(bg).  Samples are kept so that repropagate() can be replayed with a new gyroscope bias.
struct Preint {
    Vec3 lin_acc, lin_gyr;  // linearized_acc / linearized_gyr (the sample the integration starts from)
    std::vector<double> dt;
    std::vector<Vec3> acc, gyr;
    Vec3 ba, bg;
    double sum_dt = 0;
    Vec3 dp, dv;
    Quat dq;
    Mat3 J_R_bg;  // jacobian.block<3,3>(O_R, O_BG)
    Vec3 acc_0, gyr_0;
    bool valid = false;
    void start(const Vec3& a0, const Vec3& g0, const Vec3& ba_, const Vec3& bg_);
    void push_back(double dt_, const Vec3& a, const Vec3& g);
    void repropagate(const Vec3& ba_, const Vec3& bg_);

private:
    void propagate(double dt_, const Vec3& a1, const Vec3& g1);
};

struct ImageFrame {  // initial/initial_alignment.h:13-28
    double t = 0;
    std::vector<int> ids;       // ascending (std::map order)
    std::vector<double> xy;     // normalised image coordinates, 2 per id
    Mat3 R;
    Vec3 T;
    Preint pre;                 // pre.valid == false for the very first image
    bool is_key_frame = false;
};

struct Track {  // FeatureManager::feature entry reduced to what the SfM reads
    int id = 0, start_frame = 0;
    std::vector<double> xy;  // 2 per observed window frame, consecutive frames from start_frame
};

struct Result {
    int code = 0;     // 0 ok, otherwise the stage that failed (see INIT_FAIL_*)
    int l = -1;       // reference frame chosen by relativePose
    double scale = 0;
    Vec3 g;           // refined gravity in the c0 frame (before the yaw alignment of visualInitialAlign)
    Vec3 delta_bg;
    std::vector<Vec3> frame_vel;  // per all-image frame: velocity in its body frame (x.segment<3>(3 k))
    int sfm_iterations = 0;
    double sfm_cost = 0;
};

enum { INIT_OK = 0, INIT_FAIL_RELATIVE_POSE = 1, INIT_FAIL_SFM = 2, INIT_FAIL_PNP = 3, INIT_FAIL_ALIGN = 4 };

// cv::findFundamentalMat(FM_RANSAC, 0.3/460, 0.99) + cv::recoverPose with K = I on float correspondences
// (solve_5pts.cpp:193-227).  R, T are the reference's outputs (Rotation = R^T, Translation = -R^T t); returns
// inlier_cnt > 12.
bool solve_relative_rt(const std::vector<double>& corres4, Mat3& R, Vec3& T, int* inliers = nullptr);

// cv::recoverPose(E, p1, p2, I, R, t, mask): cheirality vote over the four decompositions (distance threshold 50).
int recover_pose(const double E[9], const float* p1, const float* p2, int n, unsigned char* mask, Mat3& R, Vec3& t);

// cv::solvePnP(obj, img, I, no distortion, rvec, tvec, useExtrinsicGuess = true, SOLVEPNP_ITERATIVE): Levenberg-Marquardt
// on the reprojection error from the given pose; points pass through float like cv::Point3f / cv::Point2f.
bool solve_pnp(const std::vector<double>& pts3, const std::vector<double>& pts2, Mat3& R, Vec3& t);

// GlobalSFM::triangulatePoint (initial_sfm.cpp:5-20); poses are 3x4 row major.
Vec3 triangulate_point(const double P0[12], const double P1[12], const double x0[2], const double x1[2]);

// GlobalSFM::construct.  q/T: camera-to-world rotation / position per window frame (outputs).  function_tolerance is Ceres'
// default; tests tighten it to compare the bundle's fixed point with an independent solver.
bool sfm_construct(int frame_num, std::vector<Quat>& q, std::vector<Vec3>& T, int l, const Mat3& relative_R,
                   const Vec3& relative_T, const std::vector<Track>& tracks, std::map<int, Vec3>& sfm_tracked_points,
                   int* iterations = nullptr, double* final_cost = nullptr, double function_tolerance = 1e-6);

// VisualIMUAlignment (initial_aligment.cpp:199-207): updates Bgs (all W + 1 get delta_bg), repropagates every frame's
// pre-integration with (0, Bgs[0]), solves velocities / gravity / scale.  x = [v_0 .. v_{n-1}, (g refined: 2), s].
bool visual_imu_alignment(std::vector<ImageFrame>& frames, std::vector<Vec3>& Bgs, const Vec3& tic, double g_norm, Vec3& g,
                          std::vector<double>& x, Vec3* delta_bg = nullptr);

// Estimator::relativePose (estimator.cpp:442-471) on the feature tracks of the window.
bool relative_pose(const std::vector<Track>& tracks, int window_size, Mat3& R, Vec3& T, int& l);

// initialStructure() up to and including VisualIMUAlignment: fills R/T/is_key_frame of every frame (R already multiplied
// by RIC^T as the reference stores it), Bgs, g and the alignment vector.
Result initial_structure(std::vector<ImageFrame>& frames, const std::vector<double>& headers, const std::vector<Track>& tracks,
                         const Mat3& ric, const Vec3& tic, double g_norm, std::vector<Vec3>& Bgs, std::vector<double>& x,
                         double function_tolerance = 1e-6);

// Utility::g2R (utility/utility.cpp:3-13)
Mat3 g2R(const Vec3& g);

// InitialEXRotation (initial/initial_ex_rotation.{h,cpp}): ESTIMATE_EXTRINSIC == 2, the camera-IMU rotation from pairs of
// (camera rotation out of the essential matrix of consecutive frames, gyroscope rotation delta_q of the same interval):
// q_imu (x) q_ic = q_ic (x) q_cam stacked into a 4N x 4 system with Huber weights, smallest right singular vector.
struct ExRotation {
    int frame_count = 0;
    std::vector<Mat3> Rc{Mat3()}, Rimu{Mat3()}, Rc_g{Mat3()};
    Mat3 ric;
    double last_cov1 = 0;  // second smallest singular value of the last system (the observability test: > 0.25)
    // CalibrationExRotation(corres, delta_q_imu, calib_ric_result): corres4 = n x (x0 y0 x1 y1) between the two newest frames
    // (rc_given: tests hand the camera rotation in instead of extracting it from the correspondences)
    bool calibrate(const std::vector<double>& corres4, const Quat& delta_q_imu, int window_size, Mat3& calib_ric_result,
                   const Mat3* rc_given = nullptr);
    Mat3 solve_relative_r(const std::vector<double>& corres4) const;
};

}  // namespace init
}  // namespace vb
