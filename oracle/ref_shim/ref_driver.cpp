// ref_driver.cpp — C entry points around the reference's own pose code (oracle/_ref/libplstvo_ref.so).
//
// TEST INFRASTRUCTURE.  OURS: marshalling between the plain-C structs of include/plstvo.h and the reference's classes,
// nothing else.  The numerical code is the reference's text, included below from oracle/_ref/extracted_*.inc (written by
// oracle/make_ref.py from /root/reference by line range, never committed).  Entry points mirror oracle/plstvo_oracle.h
// (orc_* -> ref_*) so tests/test_oracle_ref.py can feed both the same inputs.
#include <cstdint>
#include <cstdlib>
#include <sstream>
#include <string>

#include "stvo_standin.h"
#include "include/plstvo.h"

// ---- the reference's text ---------------------------------------------------------------------------------------------
#include "extracted_aux.inc"
#include "extracted_cam.inc"
namespace StVO {
#include "extracted_frame.inc"
#include "extracted_handler.inc"
// dead in the reference (mode is hard-wired to 0, src/stereoFrameHandler.cpp:329); never reached
void StereoFrameHandler::levenbergMarquardtOptimization(Matrix4d&, Matrix6d&, double&, int) { abort(); }
}  // namespace StVO

using namespace StVO;

namespace {

Matrix4d m4(const double* a) { Matrix4d m; for (int i = 0; i < 16; ++i) m.d_[i] = a[i]; return m; }
Matrix6d m6(const double* a) { Matrix6d m; for (int i = 0; i < 36; ++i) m.d_[i] = a[i]; return m; }
void out(const M& m, double* a) { for (int i = 0; i < m.size(); ++i) a[i] = m.d_[i]; }   // both row-major

struct Quiet {   // the reference prints from inside the GN loop and the gate; keep the test logs clean
    std::streambuf* old;
    std::ostringstream sink;
    Quiet() : old(std::cout.rdbuf(sink.rdbuf())) {}
    ~Quiet() { std::cout.rdbuf(old); }
};

void set_config(const PlConfig* cfg) {
    Config::hasPoints() = cfg->has_points != 0;
    Config::hasLines() = cfg->has_lines != 0;
    Config::useMotionModel() = cfg->use_motion_model != 0;
    Config::homogTh() = cfg->homog_th;
    Config::minFeatures() = cfg->min_features;
    Config::maxIters() = cfg->max_iters;
    Config::maxItersRef() = cfg->max_iters_ref;
    Config::minError() = cfg->min_error;
    Config::minErrorChange() = cfg->min_error_change;
    Config::inlierK() = cfg->inlier_k;
}

struct Problem {
    PinholeStereoCamera cam;
    StereoFrame prev, curr;
    StereoFrameHandler h;
    std::vector<PointFeature> pts;
    std::vector<LineFeature> lns;
    Problem(const PlCamera* c, const PlConfig* cfg, const PlMatchedBatch* m, int p) {
        set_config(cfg);
        cam.fx = c->fx; cam.fy = c->fy; cam.cx = c->cx; cam.cy = c->cy; cam.b = c->b;
        cam.width = c->width; cam.height = c->height;
        const int p0 = m->pt_off[p], p1 = m->pt_off[p + 1], l0 = m->ls_off[p], l1 = m->ls_off[p + 1];
        pts.resize(p1 - p0);
        lns.resize(l1 - l0);
        for (int i = 0; i < p1 - p0; ++i) {
            PointFeature& q = pts[i];
            for (int k = 0; k < 3; ++k) q.P(k) = m->pt_P[3 * (size_t)(p0 + i) + k];
            for (int k = 0; k < 2; ++k) q.pl_obs(k) = m->pt_pl_obs[2 * (size_t)(p0 + i) + k];
            q.pl = q.pl_obs;
            q.sigma2 = m->pt_sigma2[p0 + i];
            q.inlier = m->pt_inlier ? m->pt_inlier[p0 + i] != 0 : true;
            q.covP_an = Matrix3d::Zero();
            q.idx = i; q.level = 0; q.disp = 0.0;
            h.matched_pt.push_back(&q);
        }
        for (int i = 0; i < l1 - l0; ++i) {
            LineFeature& q = lns[i];
            for (int k = 0; k < 3; ++k) {
                q.sP(k) = m->ls_sP[3 * (size_t)(l0 + i) + k];
                q.eP(k) = m->ls_eP[3 * (size_t)(l0 + i) + k];
                q.le_obs(k) = m->ls_le_obs[3 * (size_t)(l0 + i) + k];
            }
            for (int k = 0; k < 2; ++k) {
                q.spl(k) = m->ls_spl[2 * (size_t)(l0 + i) + k];
                q.epl(k) = m->ls_epl[2 * (size_t)(l0 + i) + k];
            }
            q.le = q.le_obs;
            q.sigma2 = m->ls_sigma2[l0 + i];
            q.inlier = m->ls_inlier ? m->ls_inlier[l0 + i] != 0 : true;
            q.idx = i; q.level = 0;
            h.matched_ls.push_back(&q);
        }
        h.cam = &cam;
        h.prev_frame = &prev;
        h.curr_frame = &curr;
        // f2fTracking: n_inliers_* = list sizes (src/stereoFrameHandler.cpp:126-128)
        h.n_inliers_pt = (int)pts.size();
        h.n_inliers_ls = (int)lns.size();
        h.n_inliers = h.n_inliers_pt + h.n_inliers_ls;
        prev.Tfw = Matrix4d::Identity();
        prev.Tfw_cov = Matrix6d::Identity();   // initialize(): Tfw = I, Tfw_cov = I (src/stereoFrameHandler.cpp:43-44)
        prev.DT = Matrix4d::Identity();
        prev.DT_cov = Matrix6d::Zero();
        prev.err_norm = -1.0;
    }
    void set_prior(const PlPrior* pr) {
        if (!pr) { Config::useMotionModel() = false; return; }
        prev.Tfw = m4(pr->Tfw);
        prev.Tfw_cov = m6(pr->Tfw_cov);
        prev.DT = m4(pr->DT);
        prev.DT_cov = m6(pr->DT_cov);
        prev.err_norm = pr->err_norm;
    }
};

// optimizePose's control flow with `mode` = 1 (the reference hard-wires 0, src/stereoFrameHandler.cpp:329, so this branch
// cannot be reached through the extracted optimizePose): the flow below is OURS, every function it calls is the reference's.
void optimize_pose_mode1(Problem& q) {
    StereoFrameHandler& h = q.h;
    Matrix4d DT, DT_;
    Matrix6d DT_cov = Matrix6d::Zero();
    double err = -1.0;
    if (Config::useMotionModel()) {
        DT = q.prev.DT;
        if (!h.isGoodSolution(DT, q.prev.DT_cov, q.prev.err_norm)) DT = Matrix4d::Identity();
    } else
        DT = Matrix4d::Identity();
    if (h.n_inliers >= Config::minFeatures()) {
        DT_ = DT;
        h.gaussNewtonOptimizationRobust(DT_, DT_cov, err, Config::maxIters());
        if (h.isGoodSolution(DT_, DT_cov, err)) {
            h.removeOutliers(DT_);
            if (h.n_inliers >= Config::minFeatures()) h.gaussNewtonOptimizationRobust(DT, DT_cov, err, Config::maxItersRef());
            else DT = Matrix4d::Identity();
        } else
            h.gaussNewtonOptimizationRobust(DT, DT_cov, err, Config::maxItersRef());
    } else
        DT = Matrix4d::Identity();
    if (h.isGoodSolution(DT, DT_cov, err) && DT != Matrix4d::Identity()) {
        q.curr.DT = expmap_se3(logmap_se3(inverse_se3(DT)));
        q.curr.DT_cov = DT_cov;
        q.curr.err_norm = err;
        q.curr.Tfw = expmap_se3(logmap_se3(q.prev.Tfw * q.curr.DT));
        q.curr.Tfw_cov = unccomp_se3(q.prev.Tfw, q.prev.Tfw_cov, DT_cov);
        SelfAdjointEigenSolver<Matrix6d> es(DT_cov);
        q.curr.DT_cov_eig = es.eigenvalues();
    } else {
        q.curr.DT = Matrix4d::Identity();
        q.curr.DT_cov = Matrix6d::Zero();
        q.curr.err_norm = -1.0;
        q.curr.Tfw = q.prev.Tfw;
        q.curr.Tfw_cov = q.prev.Tfw_cov;
        q.curr.DT_cov_eig = Vector6d::Zero();
    }
}

}  // namespace

extern "C" {

const char* ref_describe() {
    return "rubengooj/stvo-pl pose path compiled from /root/reference line ranges against oracle/ref_shim stand-in headers";
}

void ref_inverse_se3(const double T[16], double Tinv[16]) { out(inverse_se3(m4(T)), Tinv); }
void ref_expmap_se3(const double x[6], double T[16]) {
    Vector6d v;
    for (int i = 0; i < 6; ++i) v(i) = x[i];
    out(expmap_se3(v), T);
}
void ref_logmap_se3(const double T[16], double x[6]) { out(logmap_se3(m4(T)), x); }
void ref_adjoint_se3(const double T[16], double Ad[36]) { out(adjoint_se3(m4(T)), Ad); }
void ref_unccomp_se3(const double T1[16], const double c1[36], const double cinc[36], double o[36]) {
    out(unccomp_se3(m4(T1), m6(c1), m6(cinc)), o);
}
int ref_is_finite(const double* x, int n) {
    MatrixXd m(n, 1);
    for (int i = 0; i < n; ++i) m.d_[i] = x[i];
    return is_finite(m) ? 1 : 0;
}
void ref_vector_mean_stdv_mad(const double* res, int n, double* mean, double* stdv) {
    vector<double> v(res, res + n);
    vector_mean_stdv_mad(v, *mean, *stdv);
}
double ref_vector_stdv_mad(const double* res, int n) {
    vector<double> v(res, res + n);
    return vector_stdv_mad(v);
}
double ref_robust_weight_cauchy(double r) { return robustWeightCauchy(r); }
double ref_line_segment_overlap(const double a[2], const double b[2], const double c[2], const double d[2]) {
    StereoFrame f;
    return f.lineSegmentOverlap(Vector2d(a[0], a[1]), Vector2d(b[0], b[1]), Vector2d(c[0], c[1]), Vector2d(d[0], d[1]));
}
void ref_projection(const PlCamera* c, const double P[3], double uv[2]) {
    PinholeStereoCamera cam;
    cam.fx = c->fx; cam.fy = c->fy; cam.cx = c->cx; cam.cy = c->cy; cam.b = c->b;
    out(cam.projection(Vector3d(P[0], P[1], P[2])), uv);
}
void ref_back_projection(const PlCamera* c, double u, double v, double disp, double P[3]) {
    PinholeStereoCamera cam;
    cam.fx = c->fx; cam.fy = c->fy; cam.cx = c->cx; cam.cy = c->cy; cam.b = c->b;
    out(cam.backProjection(u, v, disp), P);
}

// the stand-in's dense algebra, exposed so the tests can hold it against LAPACK
int ref_qr6_solve(const double H[36], const double g[6], double x[6], double* log_abs_det) {
    ColPivHouseholderQR<Matrix6d> s(m6(H));
    Vector6d b;
    for (int i = 0; i < 6; ++i) b(i) = g[i];
    out(s.solve(b), x);
    if (log_abs_det) *log_abs_det = s.logAbsDeterminant();
    return s.rank();
}
void ref_inv6(const double A[36], double Ainv[36]) { out(m6(A).inverse(), Ainv); }
void ref_eig6_sym(const double A[36], double w[6]) {
    SelfAdjointEigenSolver<Matrix6d> es(m6(A));
    out(es.eigenvalues(), w);
}

void ref_optimize_functions(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* m, int p, const double DT[16],
                            int robust, double H[36], double g[6], double* e) {
    Quiet quiet;
    Problem q(cam, cfg, m, p);
    Matrix6d Hm;
    Vector6d gm;
    double err = 0.0;
    if (robust) q.h.optimizeFunctionsRobust(m4(DT), Hm, gm, err);
    else q.h.optimizeFunctions(m4(DT), Hm, gm, err);
    out(Hm, H);
    out(gm, g);
    *e = err;
}

// one call of gaussNewtonOptimization[Robust] from DT0
void ref_gauss_newton(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* m, int p, const double DT0[16], int robust,
                      int max_iters, double DT[16], double DT_cov[36], double* err) {
    Quiet quiet;
    Problem q(cam, cfg, m, p);
    Matrix4d T = m4(DT0);
    Matrix6d C = Matrix6d::Zero();
    double e = -1.0;
    if (robust) q.h.gaussNewtonOptimizationRobust(T, C, e, max_iters);
    else q.h.gaussNewtonOptimization(T, C, e, max_iters);
    out(T, DT);
    out(C, DT_cov);
    *err = e;
}

// removeOutliers at pose DT: flags out, counts = {n_inliers_pt, n_inliers_ls, n_inliers}
int ref_remove_outliers(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* m, int p, const double DT[16],
                        uint8_t* inlier_pt, uint8_t* inlier_ls, int32_t counts[3]) {
    Quiet quiet;
    Problem q(cam, cfg, m, p);
    try {
        q.h.removeOutliers(m4(DT));
    } catch (const std::exception&) {
        return PLSTVO_E_SIZE;
    }
    for (size_t i = 0; i < q.pts.size(); ++i) inlier_pt[i] = q.pts[i].inlier;
    for (size_t i = 0; i < q.lns.size(); ++i) inlier_ls[i] = q.lns[i].inlier;
    counts[0] = q.h.n_inliers_pt; counts[1] = q.h.n_inliers_ls; counts[2] = q.h.n_inliers;
    return 0;
}

// StereoFrameHandler::optimizePose on explicit matched lists; same contract as orc_optimize_pose for the fields the
// reference exposes (iteration counts, status and DT_opt are not observable there and are left zero)
int ref_optimize_pose(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* matched, const PlPrior* priors,
                      PlPoseResult* results, uint8_t* inlier_pt, uint8_t* inlier_ls) {
    Quiet quiet;
    int rc = 0;
    for (int p = 0; p < matched->B; ++p) {
        Problem q(cam, cfg, matched, p);
        q.set_prior(priors ? &priors[p] : nullptr);
        try {
            if (cfg->solver_mode == 1) optimize_pose_mode1(q);
            else q.h.optimizePose();
        } catch (const std::exception&) {
            rc = PLSTVO_E_SIZE;
        }
        PlPoseResult& r = results[p];
        memset(&r, 0, sizeof(r));
        out(q.curr.DT, r.DT);
        out(q.curr.DT_cov, r.DT_cov);
        out(q.curr.DT_cov_eig, r.DT_cov_eig);
        r.err_norm = q.curr.err_norm;
        out(q.curr.Tfw, r.Tfw);
        out(q.curr.Tfw_cov, r.Tfw_cov);
        r.n_matched_pt = (int)q.pts.size();
        r.n_matched_ls = (int)q.lns.size();
        r.n_inliers_pt = q.h.n_inliers_pt;
        r.n_inliers_ls = q.h.n_inliers_ls;
        r.n_inliers = q.h.n_inliers;
        r.good = q.curr.err_norm != -1.0;
        if (inlier_pt)
            for (size_t i = 0; i < q.pts.size(); ++i) inlier_pt[matched->pt_off[p] + i] = q.pts[i].inlier;
        if (inlier_ls)
            for (size_t i = 0; i < q.lns.size(); ++i) inlier_ls[matched->ls_off[p] + i] = q.lns[i].inlier;
    }
    return rc;
}

// StereoFrameHandler::needNewKF on one frame (Tfw, DT, DT_cov) from the handler state s, then currFrameIsKF where it fires;
// s comes back as the handler's SLAM variables stand after both.  The function keeps its diagnostics in locals and only
// prints them, so they are read back from its own cout line, printed at 17 significant digits (round-trip exact): o gets the
// decision, N_prevKF_currF as needNewKF leaves it, and entropy_ratio, t, r; entropy_curr only where it does not fire (the
// firing line leaves it out; NaN there).  Tfw_out / Tfw_cov_out (each may be NULL): the frame's Tfw, Tfw_cov afterwards
// (Tfw_cov enters as zero).
int ref_need_new_kf(const PlKeyframeConfig* k, PlKeyframeState* s, const double Tfw[16], const double DT[16],
                    const double DT_cov[36], PlKeyframeResult* o, double Tfw_out[16], double Tfw_cov_out[36]) {
    Config::minEntropyRatio() = k->min_entropy_ratio;
    Config::maxKFTDist() = k->max_kf_t_dist;
    Config::maxKFRDist() = k->max_kf_r_dist;
    StereoFrame f;
    f.Tfw = m4(Tfw);
    f.DT = m4(DT);
    f.DT_cov = m6(DT_cov);
    f.Tfw_cov = Matrix6d::Zero();
    StereoFrameHandler h;
    h.curr_frame = &f;
    h.prev_f_iskf = s->prev_f_iskf != 0;
    h.entropy_first_prevKF = s->entropy_first_prevKF;
    h.T_prevKF = m4(s->T_prevKF);
    h.cov_prevKF_currF = m6(s->cov_prevKF_currF);
    h.N_prevKF_currF = s->N_prevKF_currF;
    bool kf;
    std::string line;
    {
        Quiet quiet;
        const std::streamsize prec = std::cout.precision(17);
        kf = h.needNewKF();
        std::cout.precision(prec);
        line = quiet.sink.str();
    }
    o->new_kf = kf ? 1 : 0;
    o->N_prevKF_currF = h.N_prevKF_currF;
    // "Entropy ratio: ratio\tt r N" or "No new KF needed: ratio\tentropy_curr entropy_first det\tt r N"
    const size_t colon = line.find(':');
    if (colon == std::string::npos) return PLSTVO_E_INVALID;
    std::istringstream in(line.substr(colon + 1));
    std::vector<double> v;
    for (std::string tok; in >> tok;) v.push_back(std::strtod(tok.c_str(), nullptr));
    if (v.size() != (kf ? 4u : 7u)) return PLSTVO_E_INVALID;
    o->entropy_ratio = v[0];
    o->entropy_curr = kf ? std::numeric_limits<double>::quiet_NaN() : v[1];
    o->t = v[kf ? 1 : 4];
    o->r = v[kf ? 2 : 5];
    if (kf) h.currFrameIsKF();
    s->prev_f_iskf = h.prev_f_iskf ? 1 : 0;
    s->entropy_first_prevKF = h.entropy_first_prevKF;
    out(h.T_prevKF, s->T_prevKF);
    out(h.cov_prevKF_currF, s->cov_prevKF_currF);
    s->N_prevKF_currF = h.N_prevKF_currF;
    if (Tfw_out) out(f.Tfw, Tfw_out);
    if (Tfw_cov_out) out(f.Tfw_cov, Tfw_cov_out);
    return 0;
}

}  // extern "C"
