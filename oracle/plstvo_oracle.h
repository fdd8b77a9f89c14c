/*
 * plstvo_oracle.h — CPU ORACLE for the PL-StVO frame-to-frame hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 * The product library (stvo_pl_b200/csrc) never includes, links or calls this code.
 *
 * It is a dependency-free restatement (plain C, double precision, scalar loops in the
 * reference's own order) of rubengooj/stvo-pl @ baecb5f; each function cites the lines it follows.
 *
 * PARITY PINNING
 *   matching half : pinned against OpenCV's cv::BFMatcher (the third-party library the
 *                   reference calls at src/matching.cpp:47-48; opencv-python 4.13.0 in this
 *                   image) through committed golden vectors, tests/golden/match_*.npz.
 *   pose half     : pinned against the reference's OWN code: oracle/make_ref.py cuts optimizeFunctions[Robust],
 *                   gaussNewtonOptimization[Robust], removeOutliers, isGoodSolution, optimizePose, lineSegmentOverlap,
 *                   projection, the SE(3) helpers and the MAD statistics verbatim out of /root/reference by line range
 *                   and compiles them against stand-in Eigen headers (oracle/ref_shim/) into oracle/_ref/;
 *                   tests/test_oracle_ref.py holds every pose function of this file against that library (identical
 *                   inlier flags, poses to 1e-9 rad / 1e-8 m, all branches).  Not Eigen's: the 6x6 decompositions
 *                   inside that library are the stand-in's (checked against LAPACK), see DESIGN.md section 4.
 */
#ifndef PLSTVO_ORACLE_H_
#define PLSTVO_ORACLE_H_

#include "../include/plstvo.h"

#ifdef __cplusplus
extern "C" {
#endif

/* src/matching.cpp:93-109 */
int orc_distance(const uint8_t* a, const uint8_t* b);
/* src/matching.cpp:41-61 (+ OpenCV BFMatcher::knnMatch semantics) */
int orc_match_nnr(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnr, int32_t* m12);
/* src/matching.cpp:63-91; threads != 0 runs both directions on two threads (lrInParallel) */
int orc_match(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnr, int best_lr,
              int threads, int32_t* m12);
/* raw 2-NN lists, for the comparison with cv2.BFMatcher: idx[2*i+k], dist[2*i+k]; -1 when absent */
void orc_knn2(const uint8_t* d1, int n1, const uint8_t* d2, int n2, int32_t* idx, int32_t* dist);

/* StVO::matchGrid, points and lines (src/matching.cpp:111-177, :179-258) with GridStructure (src/gridStructure.cpp:43-76)
 * and LineIterator (src/lineIterator.cpp:34-77) restated; one frame per call */
int orc_match_grid_points(int rows, int cols, PlGridWindow w, int best_lr, double ratio, const int32_t* q_cell,
                          const uint8_t* d1, int n1, const int32_t* t_cell, const uint8_t* d2, int n2, int32_t* m12);
int orc_match_grid_lines(int rows, int cols, PlGridWindow w, int best_lr, double ratio, double line_sim_th,
                         const int32_t* q_line, const uint8_t* d1, int n1, const double* t_line, const double* t_dir,
                         const uint8_t* d2, int n2, int32_t* m12);
/* getLineCoords: cells visited by LineIterator; returns the count, writes up to cap (x, y) pairs */
int orc_line_cells(double x1, double y1, double x2, double y2, int32_t* cells, int cap);

/* 3-D lifting of the stereo matches, one frame per call (src/stereoFrame.cpp:149-172, :348-397, :405-415, :473-508);
 * outputs dense from element 0; returns the number of surviving features */
int orc_stereo_lift_points(const PlCamera* cam, const PlStereoConfig* sc, int n_l, const float* kp_l, const int32_t* octave_l,
                           const uint8_t* desc_l, const float* kp_r, const int32_t* m12, double* pt_pl, double* pt_disp,
                           double* pt_P, double* pt_sigma2, int32_t* pt_level, uint8_t* pdesc_out, int32_t* src_idx);
int orc_stereo_lift_lines(const PlCamera* cam, const PlStereoConfig* sc, int n_l, const float* seg_l, const float* angle_l,
                          const int32_t* octave_l, const uint8_t* desc_l, const float* seg_r, const int32_t* m12,
                          double* ls_spl, double* ls_epl, double* ls_sdisp, double* ls_edisp, double* ls_sP, double* ls_eP,
                          double* ls_le, double* ls_angle, double* ls_sigma2, int32_t* ls_level, uint8_t* ldesc_out,
                          int32_t* src_idx);
/* StereoFrame::matchStereoPoints / matchStereoLines for one frame (src/stereoFrame.cpp:120-173, :309-398): grid coordinates as
 * the caller forms them (:47-48, :129-139, :318-337), matchGrid, lifting.  Outputs as orc_stereo_lift_*; m12 has n_l entries. */
int orc_match_stereo_points(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int n_l, const float* kp_l,
                            const int32_t* octave_l, const uint8_t* desc_l, int n_r, const float* kp_r, const uint8_t* desc_r,
                            int32_t* m12, double* pt_pl, double* pt_disp, double* pt_P, double* pt_sigma2, int32_t* pt_level,
                            uint8_t* pdesc_out, int32_t* src_idx);
int orc_match_stereo_lines(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int n_l, const float* seg_l,
                           const float* angle_l, const int32_t* octave_l, const uint8_t* desc_l, int n_r, const float* seg_r,
                           const uint8_t* desc_r, int32_t* m12, double* ls_spl, double* ls_epl, double* ls_sdisp, double* ls_edisp,
                           double* ls_sP, double* ls_eP, double* ls_le, double* ls_angle, double* ls_sigma2, int32_t* ls_level,
                           uint8_t* ldesc_out, int32_t* src_idx);
/* both of the above for B frames on `threads` host threads, one frame per thread at a time (the all-cores CPU baseline of
 * bench.py --workload stereo); counts[2 * f], [2 * f + 1] = lifted points, lines of frame f; records are discarded */
int orc_stereo_batch(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int B, const int32_t* pl_off,
                     const float* kp_l, const int32_t* poct_l, const uint8_t* pdesc_l, const int32_t* pr_off, const float* kp_r,
                     const uint8_t* pdesc_r, const int32_t* ll_off, const float* seg_l, const float* angle_l, const int32_t* loct_l,
                     const uint8_t* ldesc_l, const int32_t* lr_off, const float* seg_r, const uint8_t* ldesc_r, int threads,
                     int32_t* counts);
double orc_line_segment_overlap_stereo(const PlStereoConfig* sc, double spl_obs, double epl_obs, double spl_proj, double epl_proj);

/* src/auxiliar.cpp */
void   orc_inverse_se3(const double T[16], double Tinv[16]);            /* :113-122 */
void   orc_expmap_se3(const double x[6], double T[16]);                 /* :124-141 */
void   orc_logmap_se3(const double T[16], double x[6]);                 /* :143-173 */
void   orc_adjoint_se3(const double T[16], double Ad[36]);              /* :175-182 */
void   orc_unccomp_se3(const double T1[16], const double c1[36], const double cinc[36], double out[36]); /* :192-197 */
int    orc_is_finite(const double* x, int n);                           /* :353-355 */
int    orc_is_good_solution(const double DT[16], const double DT_cov[36], double err);   /* isGoodSolution, :292-305 */
void   orc_vector_mean_stdv_mad(const double* res, int n, double* mean, double* stdv); /* :387-430 */
double orc_vector_stdv_mad(const double* res, int n);                   /* :444-460 */
double orc_robust_weight_cauchy(double r);                              /* :556-559 */
/* src/stereoFrame.cpp:510-616 */
double orc_line_segment_overlap(const double spl_obs[2], const double epl_obs[2],
                                const double spl_proj[2], const double epl_proj[2]);
/* src/pinholeStereoCamera.cpp:221-237 */
void   orc_projection(const PlCamera* cam, const double P[3], double uv[2]);
void   orc_back_projection(const PlCamera* cam, double u, double v, double disp, double P[3]);

/* Eigen pieces restated numerically (agree to rounding, not bitwise) */
int    orc_qr6_solve(const double H[36], const double g[6], double x[6], double* log_abs_det); /* ColPivHouseholderQR::solve */
void   orc_inv6(const double A[36], double Ainv[36]);                   /* Matrix6d::inverse (PartialPivLU) */
void   orc_eig6_sym(const double A[36], double w[6]);                   /* SelfAdjointEigenSolver::eigenvalues, lower triangle, ascending */

/* src/stereoFrameHandler.cpp:549-694 / :696-962 on explicit lists (problem p of the batch);
 * H row-major 6x6 */
void   orc_optimize_functions(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* m, int p,
                              const double DT[16], int robust, double H[36], double g[6], double* e);

/* src/stereoFrameHandler.cpp:307-392 on explicit matched lists */
int orc_optimize_pose(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* matched,
                      const PlPrior* priors, PlPoseResult* results, uint8_t* inlier_pt,
                      uint8_t* inlier_ls);
/* src/stereoFrameHandler.cpp:106-180 */
int orc_f2f_tracking(const PlConfig* cfg, const PlFrameBatch* prev, const PlFrameBatch* curr,
                     int32_t* m12_pt, int32_t* m12_ls, int32_t* n_matched);
/* insertStereoPair's f2fTracking + optimizePose for B pairs (same contract as plstvo_track_batch).
 * threads: number of worker threads, one pair per thread at a time (all-cores throughput);
 * faithful != 0: reference-faithful threading inside a pair instead (points || lines, 1->2 || 2->1:
 * src/stereoFrameHandler.cpp:113-119, src/matching.cpp:68-74), pairs processed one at a time.
 * stage_ms (optional, [2]): wall time spent in matching and in optimizePose, summed over pairs. */
int orc_track_batch(const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
                    const PlFrameBatch* curr, const PlPrior* priors, PlPoseResult* results,
                    int32_t* m12_pt, int32_t* m12_ls, uint8_t* inlier_pt, uint8_t* inlier_ls,
                    int threads, int faithful, double* stage_ms);

/* ---- host-side state machine of the handler (SURVEY 8(f)-3) ---- */
typedef struct OrcHandlerConfig {   /* src/config.cpp:40-42, :52, :72-76, :102 */
    int32_t adaptative_fast, fast_min_th, fast_max_th, fast_inc_th, fast_feat_th, orb_fast_th;
    float   fast_err_th;
    double  min_entropy_ratio, max_kf_t_dist, max_kf_r_dist;
} OrcHandlerConfig;
typedef struct OrcKfState {         /* include/stereoFrameHandler.h:81-86 */
    int32_t prev_f_iskf, N_prevKF_currF;
    double  entropy_first_prevKF, T_prevKF[16], cov_prevKF_currF[36];
    double  entropy_curr, entropy_ratio, t, r;   /* diagnostics of the last test */
} OrcKfState;
void   orc_handler_default_config(OrcHandlerConfig* c);
/* updateFrame's adaptive FAST threshold, src/stereoFrameHandler.cpp:66-86 */
int    orc_update_fast_threshold(const OrcHandlerConfig* c, int orb_fast_th, const double DT[16], double err_norm, int n_inliers_pt);
void   orc_kf_reset(OrcKfState* s);                                                     /* :48-51, :1213-1216 */
double orc_det6(const double A[36]);                                                    /* Matrix6d::determinant */
void   orc_unctinv_se3(const double T[16], const double cov[36], double out[36]);       /* src/auxiliar.cpp:184-190 */
int    orc_need_new_kf(const OrcHandlerConfig* c, OrcKfState* s, const double Tfw[16], const double DT[16],
                       const double DT_cov[36]);                                        /* :1136-1187 */

#ifdef __cplusplus
}
#endif
#endif
