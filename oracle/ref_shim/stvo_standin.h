// stvo_standin.h — declarations the extracted reference functions need in order to compile outside their project.
//
// TEST INFRASTRUCTURE (oracle/_ref).  OURS: only the members the pose path touches, with the reference's own names and
// types (include/stereoFeatures.h:30-121, include/stereoFrame.h:85-103, include/stereoFrameHandler.h:53-98,
// include/pinholeStereoCamera.h:75-88, include/config.h:39-110 of rubengooj/stvo-pl).  CV_PI is OpenCV's literal.  The function BODIES are not
// here: oracle/make_ref.py cuts them verbatim out of /root/reference into oracle/_ref/extracted_*.inc.
#pragma once
#include <iostream>
#include <limits>
#include <list>
#include <vector>

#include "eigen_standin.h"

using namespace std;
using namespace Eigen;

typedef Matrix<double, 6, 1> Vector6d;   // include/auxiliar.h:42-43
typedef Matrix<double, 6, 6> Matrix6d;

#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define CV_PI 3.1415926535897932384626433832795   // opencv2/core/cvdef.h

// ---- src/auxiliar.cpp free functions (bodies extracted) ----
Matrix3d skew(Vector3d v);
Vector3d skewcoords(Matrix3d M);
Matrix4d inverse_se3(Matrix4d T);
Matrix4d expmap_se3(Vector6d x);
Vector6d logmap_se3(Matrix4d T);
Matrix6d adjoint_se3(Matrix4d T);
Matrix6d uncTinv_se3(Matrix4d T, Matrix6d covT);
Matrix6d unccomp_se3(Matrix4d T1, Matrix6d covT1, Matrix6d covTinc);
bool is_finite(const MatrixXd x);
void vector_mean_stdv_mad(vector<double> residues, double& mean, double& stdv);
double vector_stdv_mad(vector<double> residues);
double robustWeightCauchy(double norm_res);

// the Config values the path reads; same accessor signatures as include/config.h (static, by reference; global class)
class Config {
public:
    static Config& getInstance() { static Config c; return c; }
    static bool& hasPoints() { return getInstance().has_points; }
    static bool& hasLines() { return getInstance().has_lines; }
    static bool& useMotionModel() { return getInstance().use_motion_model; }
    static double& homogTh() { return getInstance().homog_th; }
    static int& minFeatures() { return getInstance().min_features; }
    static int& maxIters() { return getInstance().max_iters; }
    static int& maxItersRef() { return getInstance().max_iters_ref; }
    static double& minError() { return getInstance().min_error; }
    static double& minErrorChange() { return getInstance().min_error_change; }
    static double& inlierK() { return getInstance().inlier_k; }
    static double& minEntropyRatio() { return getInstance().min_entropy_ratio; }
    static double& maxKFTDist() { return getInstance().max_kf_t_dist; }
    static double& maxKFRDist() { return getInstance().max_kf_r_dist; }
    bool has_points = true, has_lines = true, use_motion_model = false;
    double homog_th = 1e-7;
    int min_features = 10, max_iters = 5, max_iters_ref = 10;
    double min_error = 1e-7, min_error_change = 1e-7, inlier_k = 4.0;
    double min_entropy_ratio = 0.85, max_kf_t_dist = 5.0, max_kf_r_dist = 15.0;
};

class PinholeStereoCamera {
public:
    int width, height;
    double fx, fy, cx, cy, b;
    Vector3d backProjection(const double& u, const double& v, const double& disp);
    Vector2d projection(const Vector3d& P);
    inline const double getB() const { return b; }
    inline const double getFx() const { return fx; }
    inline const double getFy() const { return fy; }
    inline const double getCx() const { return cx; }
    inline const double getCy() const { return cy; }
};

namespace StVO {

class PointFeature {
public:
    int idx;
    Vector2d pl, pl_obs;
    double disp;
    Vector3d P;
    bool inlier;
    int level;
    double sigma2 = 1.0;
    Matrix3d covP_an;
};

class LineFeature {
public:
    int idx;
    Vector2d spl, epl, spl_obs, epl_obs;
    double sdisp, edisp, angle, sdisp_obs, edisp_obs;
    Vector3d sP, eP;
    Vector3d le, le_obs;
    bool inlier;
    int level;
    double sigma2 = 1.0;
    Matrix3d covE_an, covS_an;
};

class StereoFrame {
public:
    double lineSegmentOverlap(Vector2d spl_obs, Vector2d epl_obs, Vector2d spl_proj, Vector2d epl_proj);
    Matrix4d Tfw;
    Matrix4d DT;
    Matrix6d Tfw_cov;
    Matrix6d DT_cov;
    Vector6d DT_cov_eig;
    double err_norm;
    vector<PointFeature*> stereo_pt;
    vector<LineFeature*> stereo_ls;
};

class StereoFrameHandler {
public:
    bool isGoodSolution(Matrix4d DT, Matrix6d DTcov, double err);
    void optimizePose();
    void removeOutliers(Matrix4d DT);
    void gaussNewtonOptimization(Matrix4d& DT, Matrix6d& DT_cov, double& err_, int max_iters);
    void gaussNewtonOptimizationRobust(Matrix4d& DT, Matrix6d& DT_cov, double& err_, int max_iters);
    void levenbergMarquardtOptimization(Matrix4d& DT, Matrix6d& DT_cov, double& err_, int max_iters);   // dead in the reference (mode == 0)
    void optimizeFunctions(Matrix4d DT, Matrix6d& H, Vector6d& g, double& e);
    void optimizeFunctionsRobust(Matrix4d DT, Matrix6d& H, Vector6d& g, double& e);
    bool needNewKF();
    void currFrameIsKF();

    list<PointFeature*> matched_pt;
    list<LineFeature*> matched_ls;
    StereoFrame* prev_frame;
    StereoFrame* curr_frame;
    PinholeStereoCamera* cam;
    int n_inliers, n_inliers_pt, n_inliers_ls;

    // slam-specific variables (include/stereoFrameHandler.h:81-86)
    bool prev_f_iskf;
    double entropy_first_prevKF;
    Matrix4d T_prevKF;
    Matrix6d cov_prevKF_currF;
    int N_prevKF_currF;
};

}  // namespace StVO
