/*
 * plstvo.h — C-ABI of the H100-native PL-StVO frame-to-frame pose engine.
 *
 * Plain C, plain pointers and sizes; no Eigen / OpenCV / torch types cross this
 * boundary.  Every entry point names the reference interface it replaces
 * (paths relative to the rubengooj/stvo-pl checkout).  The reference-side
 * binding a maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions
 *  - all 4x4 / 6x6 matrices are row-major doubles (Eigen is column-major: the
 *    shim transposes on the way in/out);
 *  - descriptors are rows of exactly 32 bytes (ORB and LBD: cv::Mat N x 32
 *    CV_8UC1, continuous) — src/matching.cpp:93-109 hard-codes 8 x int32;
 *  - twist layout x = [t(3); w(3)] (src/auxiliar.cpp:124-141);
 *  - functions return >= 0 on success (a count where the reference returns
 *    one) and a negative PLSTVO_E_* code where the reference throws
 *    (src/matching.cpp:50-51, src/stereoFrameHandler.cpp:1065-1066).
 *    optimizePose never throws in the reference: failure is encoded in the
 *    result exactly as src/stereoFrameHandler.cpp:382-391 does.
 */
#ifndef PLSTVO_H_
#define PLSTVO_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PLSTVO_VERSION        100
#define PLSTVO_DESC_BYTES     32
#define PLSTVO_MAX_FEATURES   65535   /* per frame and feature type (16-bit index in the packed (dist,idx) key) */

/* error codes (negative returns) */
#define PLSTVO_E_INVALID      (-1)  /* bad argument (null pointer, negative size, stride != 32) */
#define PLSTVO_E_TOO_LARGE    (-2)  /* more than PLSTVO_MAX_FEATURES rows */
#define PLSTVO_E_CUDA         (-3)  /* CUDA runtime failure; see plstvo_last_error() */
#define PLSTVO_E_NO_DEVICE    (-4)  /* no sm_90 device: the library never falls back to a CPU path */
#define PLSTVO_E_SIZE         (-5)  /* size mismatch (the reference's std::runtime_error cases) */

/* ---- camera: PinholeStereoCamera getters used by the path
 *      (include/pinholeStereoCamera.h:80-88, src/pinholeStereoCamera.cpp:221-237) */
typedef struct PlCamera {
    double fx, fy, cx, cy, b;
    int32_t width, height;
} PlCamera;

/* ---- the ~15 Config values the path reads (include/config.h:39-105,
 *      defaults src/config.cpp:36-113, KITTI values config/config/config_kitti.yaml) */
typedef struct PlConfig {
    int32_t has_points;        /* Config::hasPoints()      */
    int32_t has_lines;         /* Config::hasLines()       */
    int32_t best_lr_matches;   /* Config::bestLRMatches()  — mutual check in StVO::match */
    int32_t use_motion_model;  /* Config::useMotionModel() */
    int32_t min_features;      /* Config::minFeatures()    */
    int32_t max_iters;         /* Config::maxIters()       */
    int32_t max_iters_ref;     /* Config::maxItersRef()    */
    int32_t solver_mode;       /* `mode` of optimizePose (src/stereoFrameHandler.cpp:329): 0 = GN (the hard-wired value), 1 = GN-robust */
    double  min_ratio_12_p;    /* narrowed to float at the call, src/stereoFrameHandler.cpp:141 */
    double  min_ratio_12_l;    /* src/stereoFrameHandler.cpp:164 */
    double  homog_th;
    double  min_error;
    double  min_error_change;
    double  inlier_k;
    double  lsd_scale;         /* Config::lsdScale(): LineFeature::safeCopy re-applies it (src/stereoFeatures.cpp:117-135) */
} PlConfig;

/* ---- a batch of B stereo frames with pre-extracted features (the contents of
 *      StereoFrame::stereo_pt / stereo_ls / pdesc_l / ldesc_l, include/stereoFrame.h:59-115),
 *      structure-of-arrays, frames concatenated; *_off are prefix sums with B+1 entries.
 *      Arrays the role does not read may be NULL:
 *        as `prev`: pdesc, ldesc, pt_P, pt_sigma2, ls_sP, ls_eP, ls_spl, ls_epl, ls_sigma2, ls_level
 *        as `curr`: pdesc, ldesc, pt_pl, ls_le                                                      */
typedef struct PlFrameBatch {
    int32_t        B;
    const int32_t* pt_off;     /* [B+1] */
    const int32_t* ls_off;     /* [B+1] */
    const uint8_t* pdesc;      /* [n_pt][32]  StereoFrame::pdesc_l */
    const uint8_t* ldesc;      /* [n_ls][32]  StereoFrame::ldesc_l */
    const double*  pt_P;       /* [n_pt][3]   PointFeature::P      (include/stereoFeatures.h:30-58) */
    const double*  pt_pl;      /* [n_pt][2]   PointFeature::pl     */
    const double*  pt_sigma2;  /* [n_pt]      PointFeature::sigma2 */
    const double*  ls_sP;      /* [n_ls][3]   LineFeature::sP      (include/stereoFeatures.h:60-121) */
    const double*  ls_eP;      /* [n_ls][3]   LineFeature::eP      */
    const double*  ls_le;      /* [n_ls][3]   LineFeature::le      */
    const double*  ls_spl;     /* [n_ls][2]   LineFeature::spl     */
    const double*  ls_epl;     /* [n_ls][2]   LineFeature::epl     */
    const double*  ls_sigma2;  /* [n_ls]      LineFeature::sigma2  */
    const int32_t* ls_level;   /* [n_ls]      LineFeature::level   */
} PlFrameBatch;

/* ---- explicit matched lists for B problems (StereoFrameHandler::matched_pt / matched_ls after
 *      f2fTracking, i.e. after safeCopy: sigma2 is used as given) */
typedef struct PlMatchedBatch {
    int32_t        B;
    const int32_t* pt_off;     /* [B+1] */
    const int32_t* ls_off;     /* [B+1] */
    const double*  pt_P;       /* [n][3] */
    const double*  pt_pl_obs;  /* [n][2] */
    const double*  pt_sigma2;  /* [n]    */
    const uint8_t* pt_inlier;  /* [n] or NULL (= all true, as f2fTracking leaves them) */
    const double*  ls_sP;      /* [m][3] */
    const double*  ls_eP;      /* [m][3] */
    const double*  ls_le_obs;  /* [m][3] */
    const double*  ls_spl;     /* [m][2] previous-frame endpoints (src/stereoFrameHandler.cpp:668) */
    const double*  ls_epl;     /* [m][2] */
    const double*  ls_sigma2;  /* [m]    */
    const uint8_t* ls_inlier;  /* [m] or NULL */
} PlMatchedBatch;

/* ---- state of prev_frame read by optimizePose (src/stereoFrameHandler.cpp:317-326, :377-378) */
typedef struct PlPrior {
    double Tfw[16];
    double Tfw_cov[36];
    double DT[16];
    double DT_cov[36];
    double err_norm;
} PlPrior;

/* status: which branch of optimizePose produced the result */
#define PLSTVO_ST_REFINED          0  /* stage 1 ok -> removeOutliers -> stage 2 (src/stereoFrameHandler.cpp:341-350) */
#define PLSTVO_ST_ROBUST_FALLBACK  1  /* stage 1 rejected -> gaussNewtonOptimizationRobust (:357-359) */
#define PLSTVO_ST_FEW_BEFORE       2  /* n_inliers < minFeatures before optimisation (:364-368) */
#define PLSTVO_ST_FEW_AFTER        3  /* n_inliers < minFeatures after removeOutliers (:351-355) */

/* ---- what optimizePose leaves in curr_frame and the handler (src/stereoFrameHandler.cpp:372-391) */
typedef struct PlPoseResult {
    double  DT[16];          /* curr_frame->DT = expmap(logmap(inverse(DT_opt)))  (:374) */
    double  DT_cov[36];      /* curr_frame->DT_cov                                (:375) */
    double  DT_cov_eig[6];   /* ascending                                        (:379-380) */
    double  err_norm;        /* curr_frame->err_norm, -1 on failure               (:376,:387) */
    double  Tfw[16];         /* curr_frame->Tfw                                   (:377,:388) */
    double  Tfw_cov[36];     /* curr_frame->Tfw_cov                               (:378,:389) */
    double  DT_opt[16];      /* the optimised prev->curr transform before inversion (diagnostic) */
    int32_t n_matched_pt;    /* matched_pt.size() */
    int32_t n_matched_ls;    /* matched_ls.size() */
    int32_t n_inliers_pt;
    int32_t n_inliers_ls;
    int32_t n_inliers;
    int32_t good;            /* 1 iff the final isGoodSolution && DT != I branch was taken (:372) */
    int32_t status;          /* PLSTVO_ST_* */
    int32_t iters_stage1;    /* evaluations of optimizeFunctions in the first GN call  */
    int32_t iters_stage2;    /* evaluations in the refinement / robust fallback call   */
    int32_t reserved;
} PlPoseResult;

typedef struct PlContext PlContext;   /* one per GPU; owns streams, device and pinned buffers */
typedef struct PlDeviceBatch PlDeviceBatch; /* inputs resident in HBM (throughput mode) */

/* ---- life cycle ------------------------------------------------------------------------------- */
int         plstvo_version(void);
/* device < 0: use the current device.  Fails with PLSTVO_E_NO_DEVICE when there is no CUDA device. */
int         plstvo_create(int device, PlContext** out);
void        plstvo_destroy(PlContext* ctx);
const char* plstvo_last_error(const PlContext* ctx);
void        plstvo_default_config(PlConfig* cfg);        /* src/config.cpp:36-113 */
void        plstvo_kitti_config(PlConfig* cfg);          /* config/config/config_kitti.yaml */

/* ---- include/matching.h surface --------------------------------------------------------------- */
/* StVO::matchNNR (src/matching.cpp:41-61): m12[i] = index of the nearest row of d2 or -1; returns #accepted.
 * The reference has undefined behaviour for n2 < 2; here every row gets -1. */
int plstvo_match_nnr(PlContext* ctx, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                     int stride_bytes, float nnr, int32_t* m12);
/* StVO::match (src/matching.cpp:63-91): matchNNR both ways + mutual filter when best_lr_matches != 0. */
int plstvo_match(PlContext* ctx, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                 int stride_bytes, float nnr, int best_lr_matches, int32_t* m12);
/* Batched form: problem p matches rows [off1[p],off1[p+1]) of d1 against [off2[p],off2[p+1]) of d2.
 * m12 holds indices local to the problem.  counts[p] (optional) = the reference's return value. */
int plstvo_match_batch(PlContext* ctx, int B, const uint8_t* d1, const int32_t* off1,
                       const uint8_t* d2, const int32_t* off2, float nnr, int best_lr_matches,
                       int32_t* m12, int32_t* counts);

/* ---- include/matching.h surface, the stereo (left/right) step: StVO::matchGrid (src/matching.cpp:111-258) ----------
 * SURVEY 8(f)-1, the row next to the hot path: same 256-bit Hamming primitive, candidates restricted to a window of
 * the 64 x 48 bucket grid (GridStructure::get, src/gridStructure.cpp:65-76), the loop-carried gate of
 * Config::bestLRMatches() (a train is only considered by a query if it beats the train's running minimum over all
 * EARLIER queries, :145-150), best / second best with multiplicity, ratio test in double, mutual filter.
 * Batched over B frames: q_off / t_off are prefix offsets of queries (left image) and trains (right image). */
typedef struct PlGridWindow {   /* GridWindow: width = (left, right), height = (up, down), include/gridStructure.h:39-41 */
    int32_t left, right, up, down;
} PlGridWindow;

/* points (src/matching.cpp:111-177; caller src/stereoFrame.cpp:129-146): q_cell / t_cell = integer grid cell (x, y) of
 * every query / train keypoint (kp.pt.x * inv_width, kp.pt.y * inv_height truncated).  m12: problem-local index or -1.
 * counts (optional) = the reference's return value per frame. */
int plstvo_match_grid_points(PlContext* ctx, int B, int grid_rows, int grid_cols, PlGridWindow w, int best_lr_matches,
                             double min_ratio_12_p, const int32_t* q_off, const int32_t* q_cell, const uint8_t* d1,
                             const int32_t* t_off, const int32_t* t_cell, const uint8_t* d2, int32_t* m12,
                             int32_t* counts);
/* lines (src/matching.cpp:179-258; caller src/stereoFrame.cpp:318-345): q_line = integer cells (sp.x, sp.y, ep.x, ep.y) of
 * the query segments; t_line = train segment end points in GRID UNITS as doubles (x1, y1, x2, y2), rasterised into
 * cells exactly like getLineCoords / LineIterator (src/lineIterator.cpp:34-77); t_dir = directions2 (normalised).
 * The reference uses minRatio12P here too (:241). */
int plstvo_match_grid_lines(PlContext* ctx, int B, int grid_rows, int grid_cols, PlGridWindow w, int best_lr_matches,
                            double min_ratio_12_p, double line_sim_th, const int32_t* q_off, const int32_t* q_line,
                            const uint8_t* d1, const int32_t* t_off, const double* t_line, const double* t_dir,
                            const uint8_t* d2, int32_t* m12, int32_t* counts);

/* ---- 3-D lifting of the stereo matches (SURVEY 8(f)-2): the step that turns matchGrid's output into the PointFeature /
 * LineFeature records the solver consumes (src/stereoFrame.cpp:149-172 points, :348-397 lines, filterLineSegmentDisparity
 * :405-415, lineSegmentOverlapStereo :473-508, backProjection src/pinholeStereoCamera.cpp:221-229).  Pure per-feature
 * arithmetic + an ordered compaction (surviving features keep ascending left index, like the reference's push_back loop).
 * Batched over B frames; outputs of frame p are written densely starting at element l_off[p]; counts[p] = survivors. */
typedef struct PlStereoConfig {   /* Config accessors read by this step (include/config.h:72-96, src/config.cpp:58-106) */
    double max_dist_epip, min_disp, ls_min_disp_ratio, line_horiz_th, stereo_overlap_th, orb_scale_factor, lsd_scale;
} PlStereoConfig;
void plstvo_default_stereo_config(PlStereoConfig* c);
/* kp_l / kp_r: cv::KeyPoint::pt (float x, y); octave_l: cv::KeyPoint::octave; m12: matchGrid output (local right index or -1).
 * out: PointFeature::pl, disp, P, sigma2, level; pdesc_out = the surviving rows of desc_l (pdesc_l_aux); src_idx = their i1. */
int plstvo_stereo_lift_points(PlContext* ctx, const PlCamera* cam, const PlStereoConfig* scfg, int B, const int32_t* l_off,
                              const float* kp_l, const int32_t* octave_l, const uint8_t* desc_l, const int32_t* r_off,
                              const float* kp_r, const int32_t* m12, double* pt_pl, double* pt_disp, double* pt_P,
                              double* pt_sigma2, int32_t* pt_level, uint8_t* pdesc_out, int32_t* src_idx, int32_t* counts);
/* seg_l / seg_r: KeyLine start / end points (float sx, sy, ex, ey); angle_l: KeyLine::angle; octave_l: KeyLine::octave.
 * out: LineFeature::spl, epl, sdisp, edisp, sP, eP, le, angle, sigma2, level; ldesc_out, src_idx as for points. */
int plstvo_stereo_lift_lines(PlContext* ctx, const PlCamera* cam, const PlStereoConfig* scfg, int B, const int32_t* l_off,
                             const float* seg_l, const float* angle_l, const int32_t* octave_l, const uint8_t* desc_l,
                             const int32_t* r_off, const float* seg_r, const int32_t* m12, double* ls_spl, double* ls_epl,
                             double* ls_sdisp, double* ls_edisp, double* ls_sP, double* ls_eP, double* ls_le,
                             double* ls_angle, double* ls_sigma2, int32_t* ls_level, uint8_t* ldesc_out, int32_t* src_idx,
                             int32_t* counts);

/* ---- StereoFrame::matchStereoPoints / matchStereoLines (src/stereoFrame.cpp:120-173, :309-398) in one device pass:
 * grid cells from the raw key points / key lines (:129-139, :318-337: x * inv_width truncated, inv_width = grid_cols / image
 * width), matchGrid, and the 3-D lifting, with the match list handed from kernel to kernel in HBM.  Inputs and outputs are
 * those of plstvo_stereo_lift_*; desc_r = right descriptors; m12 (optional) = matchGrid's list per left feature. */
typedef struct PlStereoMatchConfig {   /* include/stereoFrame.h:51-52, src/config.cpp:51, :60, :63, :91 */
    int32_t grid_rows, grid_cols;      /* GRID_ROWS 48, GRID_COLS 64 */
    int32_t matching_s_ws;             /* Config::matchingSWs(): cells to the left of the query, same row */
    int32_t best_lr_matches;
    double  min_ratio_12_p, line_sim_th;
} PlStereoMatchConfig;
void plstvo_default_stereo_match_config(PlStereoMatchConfig* c);
int plstvo_match_stereo_points(PlContext* ctx, const PlCamera* cam, const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                               int B, const int32_t* l_off, const float* kp_l, const int32_t* octave_l, const uint8_t* desc_l,
                               const int32_t* r_off, const float* kp_r, const uint8_t* desc_r, int32_t* m12, double* pt_pl,
                               double* pt_disp, double* pt_P, double* pt_sigma2, int32_t* pt_level, uint8_t* pdesc_out,
                               int32_t* src_idx, int32_t* counts);
int plstvo_match_stereo_lines(PlContext* ctx, const PlCamera* cam, const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                              int B, const int32_t* l_off, const float* seg_l, const float* angle_l, const int32_t* octave_l,
                              const uint8_t* desc_l, const int32_t* r_off, const float* seg_r, const uint8_t* desc_r,
                              int32_t* m12, double* ls_spl, double* ls_epl, double* ls_sdisp, double* ls_edisp, double* ls_sP,
                              double* ls_eP, double* ls_le, double* ls_angle, double* ls_sigma2, int32_t* ls_level,
                              uint8_t* ldesc_out, int32_t* src_idx, int32_t* counts);

/* ---- raw stereo features in, pose out: the matching half of StereoFrame::extractStereoFeatures (matchStereoPoints +
 * matchStereoLines, src/stereoFrame.cpp:120-173, :309-398) for the previous and the current frame of B independent pairs, then
 * f2fTracking + optimizePose (src/stereoFrameHandler.cpp:106-180, :307-392) on the lifted records, which never leave HBM.
 * The only host hop in between is the per-frame survivor counts (the tile plan of the descriptor matcher needs them). */
typedef struct PlStereoFeatures {      /* what detectStereoFeatures leaves for B frames (src/stereoFrame.cpp:78-118, :184-307) */
    int32_t        B;
    const int32_t* pl_off;  const int32_t* pr_off;    /* [B+1] left / right key points */
    const float*   kp_l;    const float*   kp_r;      /* [n][2] cv::KeyPoint::pt */
    const int32_t* poct_l;                            /* [n_l] cv::KeyPoint::octave */
    const uint8_t* pdesc_l; const uint8_t* pdesc_r;   /* [n][32] */
    const int32_t* ll_off;  const int32_t* lr_off;    /* [B+1] left / right key lines */
    const float*   seg_l;   const float*   seg_r;     /* [m][4] start / end point */
    const float*   angle_l;                           /* [m_l] KeyLine::angle */
    const int32_t* loct_l;                            /* [m_l] KeyLine::octave */
    const uint8_t* ldesc_l; const uint8_t* ldesc_r;   /* [m][32] */
} PlStereoFeatures;
/* n_stereo (optional): [B][4] = stereo_pt.size(), stereo_ls.size() of the previous and of the current frame. */
int plstvo_track_stereo_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                              const PlStereoConfig* scfg, const PlStereoFeatures* prev, const PlStereoFeatures* curr,
                              const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo);

/* The same for a SEQUENCE: `frames` holds B + 1 consecutive frames, pair p = (frame p, frame p + 1), B results.  Every frame goes
 * through the stereo step once (it is the current frame of one pair and the previous frame of the next, like curr_frame ->
 * prev_frame in updateFrame, src/stereoFrameHandler.cpp:98-100).  Results are per pair with priors[p] as given (NULL: identity):
 * the chaining of Tfw along the sequence (:377-378) is a host-side scan over the B results (plstvo.hpp: chainPoses).
 * n_stereo (optional): [B + 1][2] = stereo_pt.size(), stereo_ls.size() per frame. */
int plstvo_track_stereo_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                 const PlStereoConfig* scfg, const PlStereoFeatures* frames, const PlPrior* priors,
                                 PlPoseResult* results, int32_t* n_stereo);

/* Streaming forms: enqueue and return a ticket (0 / 1) like plstvo_track_batch_async; results / n_stereo are valid after
 * plstvo_wait(ctx, ticket).  Two batches may be in flight, so the next batch's uploads run under this batch's kernels; inputs
 * must stay untouched (and should be pinned, plstvo_host_alloc) until the wait returns.
 * NOT fully asynchronous: the call itself blocks (holding the context's lock) until the stereo step of this batch has run on
 * the device, because the number of lifted stereo features per frame — a result of that step — sizes the tracking plan that
 * is built on the host; what overlaps with the caller (and with the other ticket) is the tracking half and the downloads. */
int plstvo_track_stereo_batch_async(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                    const PlStereoConfig* scfg, const PlStereoFeatures* prev, const PlStereoFeatures* curr,
                                    const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo);
int plstvo_track_stereo_sequence_async(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                       const PlStereoConfig* scfg, const PlStereoFeatures* frames, const PlPrior* priors,
                                       PlPoseResult* results, int32_t* n_stereo);

/* ---- ORB description: what cv::ORB does after key-point selection (the pdesc_l / pdesc_r above) ---- */
typedef struct PlOrbConfig {       /* cv::ORB parameters; src/config.cpp:95-102 defaults */
    int32_t n_levels;              /* pyramid levels (1..32) */
    double  scale_factor;          /* level l is cvRound(W / s^l) x cvRound(H / s^l) */
    int32_t edge_threshold;        /* key points with cvRound(pt) closer than this to the border are dropped */
    int32_t patch_size;            /* 31 only */
    int32_t wta_k;                 /* 2 only */
} PlOrbConfig;
void plstvo_default_orb_config(PlOrbConfig* c);   /* 4 levels, 1.2, 19, 31, 2 */
/* Angles and 256-bit rBRIEF descriptors of given key points on n_img grey images of one size (images: [n_img][height][width]
 * uint8, row-major), bit-identical to OpenCV 4.13's ORB.  Image i's key points are rows kp_off[i] .. kp_off[i + 1] of
 * kp_xy ([n][2] float x, y in image coordinates, cv::KeyPoint::pt), kp_octave ([n]) and kp_angle ([n] degrees).
 *   kp_angle == NULL: the angle is computed (intensity centroid at cvRound(pt / scale^octave) on the octave's level), as
 *                     detectAndCompute does for its own key points;
 *   kp_angle != NULL: the angles are used as given, as ORB::compute does.
 * Key points with cvRound(pt) closer than edge_threshold to the image border are dropped (KeyPointsFilter::runByImageBorder);
 * image i's survivors, in input order, are rows kp_off[i] .. kp_off[i] + counts[i] of out_angle ([n]), out_desc ([n][32],
 * the layout PlStereoFeatures::pdesc_l / pdesc_r take) and src_idx ([n], index within the image's key points); later rows are
 * left unchanged.  Returns the number of survivors.  PLSTVO_E_INVALID: patch_size != 31, wta_k != 2, n_levels outside
 * 1..32, scale_factor <= 1 with more than one level, a level of zero size, or an octave outside [0, n_levels);
 * PLSTVO_E_TOO_LARGE: more than PLSTVO_MAX_FEATURES key points in one image. */
int plstvo_orb_compute_batch(PlContext* ctx, const PlOrbConfig* cfg, int n_img, int width, int height, const uint8_t* images,
                             const int32_t* kp_off, const float* kp_xy, const int32_t* kp_octave, const float* kp_angle,
                             float* out_angle, uint8_t* out_desc, int32_t* src_idx, int32_t* counts);
/* Device time of the last plstvo_orb_compute_batch on this context, ms: [0] pyramid and blur, [1] border filter,
 * [2] angles and descriptors. */
int plstvo_orb_kernel_times(PlContext* ctx, float* ms3);

/* ---- ORB detection + description: cv::ORB::detectAndCompute with an empty mask ---- */
typedef struct PlOrbDetectConfig {
    PlOrbConfig orb;               /* pyramid, edge threshold, patch, WTA_K (scale_factor is rounded to float, as ORB::create takes it) */
    int32_t n_features;            /* nfeatures (>= 0), spread over the levels as ORB spreads it */
    int32_t score_type;            /* 1: FAST_SCORE, 0: HARRIS_SCORE */
    int32_t fast_threshold;        /* used where fast_th == NULL; clamped to [0, 255] */
} PlOrbDetectConfig;
void plstvo_default_orb_detect_config(PlOrbDetectConfig* c);   /* 1200, 1.2, 4, 19, FAST, 31, 2, 20 */
/* Key points, angles and descriptors of n_img grey images of one size (images: [n_img][height][width] uint8), bit-identical
 * to OpenCV 4.13's ORB::detectAndCompute(image, noArray()) per image.  fast_th: [n_img] FAST thresholds, or NULL for
 * cfg->fast_threshold everywhere.  Image i's key points are rows kp_off[i] .. kp_off[i + 1] of kp_xy ([n][2], pt), kp_octave,
 * kp_angle (degrees), kp_response (FAST score or Harris response) and desc ([n][32], the layout PlStereoFeatures takes);
 * within an image they are ordered by level, then y, then x on the level (the set and every field equal OpenCV's; OpenCV's
 * order is that of nth_element).  Any of kp_xy .. desc may be NULL to skip that output.  Returns the number of key points.
 * PLSTVO_E_TOO_LARGE: more than capacity key points in all, or more than PLSTVO_MAX_FEATURES in one image; kp_off
 * ([n_img + 1]) is still written in full, so the caller can size its buffers and call again.  PLSTVO_E_INVALID: the
 * PlOrbConfig checks of plstvo_orb_compute_batch, n_features < 0, or score_type other than 0 or 1. */
int plstvo_orb_detect_and_compute_batch(PlContext* ctx, const PlOrbDetectConfig* cfg, int n_img, int width, int height,
                                        const uint8_t* images, const int32_t* fast_th, int capacity, int32_t* kp_off,
                                        float* kp_xy, int32_t* kp_octave, float* kp_angle, float* kp_response, uint8_t* desc);
/* Device time of the last plstvo_orb_detect_and_compute_batch on this context, ms: [0] pyramid and blur, [1] FAST and
 * non-max suppression, [2] selection (retainBest, Harris), [3] angles and descriptors. */
int plstvo_orb_detect_kernel_times(PlContext* ctx, float* ms4);

/* ---- LBD line description: BinaryDescriptor::compute of given key lines ---- */
/* BinaryDescriptor::compute (3rdparty/line_descriptor/src/binary_descriptor_custom.cpp:539-687, default Params: 9 bands of
 * width 7, one octave) of octave-0 key lines on n_img grey images of one size (images: [n_img][height][width] uint8),
 * bit-identical to the reference evaluated unfused.  Image i's lines are rows kl_off[i] .. kl_off[i + 1] of kl_seg ([n][4]
 * float sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY), kl_angle ([n] KeyLine::angle, radians) and
 * kl_npix ([n] KeyLine::numOfPixels); out_desc [n][32] (the layout PlStereoFeatures::ldesc_l / ldesc_r take).  Row i is
 * line i's descriptor (KeyLine::class_id is not read).  An image without lines writes nothing.  Returns the number of
 * lines.  PLSTVO_E_INVALID: a null pointer where lines exist, width or height outside 1..32767, a numOfPixels outside
 * 1..32767, or offsets that do not start at 0 or decrease; PLSTVO_E_TOO_LARGE: more than PLSTVO_MAX_FEATURES lines in one
 * image. */
int plstvo_lbd_compute_batch(PlContext* ctx, int n_img, int width, int height, const uint8_t* images, const int32_t* kl_off,
                             const float* kl_seg, const float* kl_angle, const int32_t* kl_npix, uint8_t* out_desc);
/* Device time of the last plstvo_lbd_compute_batch on this context, ms: [0] blur and Sobel, [1] descriptors. */
int plstvo_lbd_kernel_times(PlContext* ctx, float* ms2);

/* ---- LSD line detection: StereoFrame::detectLineFeatures' LSD branch (src/stereoFrame.cpp:218-241) ---- */
typedef struct PlLsdConfig {       /* Config::lsd*; src/config.cpp defaults */
    int32_t refine;                /* lsd_refine: 0 (LSD_REFINE_NONE) only */
    double  scale;                 /* lsd_scale (> 0, not 0.5): the image is blurred and resized by it before detection */
    double  sigma_scale;           /* lsd_sigma_scale (> 0) */
    double  quant;                 /* lsd_quant (>= 0) */
    double  ang_th;                /* lsd_ang_th, degrees, (0, 180) */
    int32_t n_bins;                /* lsd_n_bins, 1..4096 */
    double  min_line_length;       /* min_line_length (>= 0), relative to min(width, height) as in Config */
    int32_t n_features;            /* lsd_nfeatures (>= 0; 0 keeps every line) */
} PlLsdConfig;
void plstvo_default_lsd_config(PlLsdConfig* c);   /* 0, 1.2, 0.6, 2.0, 22.5, 1024, 0.025, 300 */
/* Key lines of n_img grey images of one size (images: [n_img][height][width] uint8), bit-identical to the reference's
 * LSDDetectorC::detect(img, lines, 1, 1, opts) on OpenCV 4.13's LineSegmentDetector followed by detectLineFeatures'
 * response sort and truncation to n_features, with min_length = min_line_length * min(width, height).  Image i's lines are
 * rows kl_off[i] .. kl_off[i + 1] of kl_seg ([n][4] float sPointInOctaveX, sPointInOctaveY, ePointInOctaveX,
 * ePointInOctaveY), kl_angle (KeyLine::angle, radians), kl_npix (numOfPixels), kl_response and kl_length (lineLength), in
 * the reference's order (class_id is the row within the image).  These are what plstvo_lbd_compute_batch and
 * PlStereoImages take.  numOfPixels is LineIterator's count after clipping to the image, so it is 0 for a line whose
 * rounded endpoints both leave the image on one side (plstvo_lbd_compute_batch rejects such a line, as it rejects any
 * numOfPixels outside 1..32767).  Any of kl_seg .. kl_length may be NULL to skip that output.  Returns the number of lines.
 * PLSTVO_E_TOO_LARGE: more than capacity lines in all, or more than PLSTVO_MAX_FEATURES in one image; kl_off ([n_img + 1]) is
 * still written in full.  PLSTVO_E_INVALID: a null config, kl_off or images, more than 65535 images, width or height outside
 * 1..32767, refine != 0,
 * a parameter outside the ranges above, a blur wider than 31 taps, or a scaled size outside 1..32767.  The whole batch is
 * resident at once: about 35 bytes of device memory per pixel of each scaled image (24 MB per 1241x376 image at scale 1.2);
 * PLSTVO_E_CUDA when that cannot be allocated. */
int plstvo_lsd_detect_batch(PlContext* ctx, const PlLsdConfig* cfg, int n_img, int width, int height, const uint8_t* images,
                            int capacity, int32_t* kl_off, float* kl_seg, float* kl_angle, int32_t* kl_npix,
                            float* kl_response, float* kl_length);
/* Device time of the last plstvo_lsd_detect_batch on this context, ms: [0] blur and resize, [1] gradient and seed order,
 * [2] region growing, [3] the host's region angles, [4] rectangles. */
int plstvo_lsd_kernel_times(PlContext* ctx, float* ms5);
/* The KeyLine step of the reference's FLD line branch (Config::useFLDLines, src/stereoFrame.cpp:260-299) for one image of
 * width x height: seg [n_seg][4] is cv::ximgproc::FastLineDetector::detect's output on fld_img, as Vec4f (start x, y, end
 * x, y), in its order.  The caller runs FLD: createFastLineDetector(min_line_length * min(width, height)) on fld_img, the
 * grey image, or for a colour image cvtColor(img, COLOR_RGB2GRAY) (the branch's CV_RGB2GRAY).  Where n_seg > n_features and
 * n_features != 0 the segments are sorted by sort_flines_by_length (include/auxiliar.h:149-154: the double
 * sqrt(pow(dx, 2.0) + pow(dy, 2.0)), strict >, libstdc++'s std::sort on the given order, so equal lengths land where the
 * reference puts them) and truncated to n_features.  Each kept segment becomes a key line, byte for byte the reference's:
 * kl_seg the segment as given (no clamp to the image: the LSD branch's checkLineExtremes does not apply), kl_length
 * (float)sqrt(pow(dx, 2) + pow(dy, 2)), kl_angle atan2 of the float differences (std::atan2(float, float), glibc's
 * atan2f), kl_response length / max(width, height), kl_npix cv::LineIterator(fld_img, start, end).count on the unclamped
 * endpoints (after LineIterator's own clipping; 0 for a segment whose rounded endpoints both leave the image on one side).
 * Such a line is returned as the reference computes it, and plstvo_lbd_compute_batch and the sessions then refuse it
 * (numOfPixels 1..32767), as the images calls do.  Any output may be NULL; the arrays hold min(n_seg, n_features) rows
 * (n_seg where n_features is 0).  Host code, no context or GPU.  Returns the number of key lines; PLSTVO_E_INVALID for
 * width or height outside 1..32767, n_features < 0, n_seg < 0, seg NULL with n_seg > 0, or a coordinate that is not finite or
 * lies outside [-2^31, 2^31) (where cvRound, which LineIterator rounds with, leaves int; FastLineDetector never gives one). */
int plstvo_fld_key_lines(int width, int height, int n_features, int n_seg, const float* seg, float* kl_seg, float* kl_angle,
                         int32_t* kl_npix, float* kl_response, float* kl_length);

/* ---- stereo images in, pose out: StereoFrame::extractStereoFeatures (src/stereoFrame.cpp:59-118, :182-243) with LSD left
 * to the caller, then matchStereoPoints / matchStereoLines, f2fTracking and optimizePose (plstvo_track_stereo_images_lsd_*
 * below run LSD too) ---- */
typedef struct PlStereoImages {
    int32_t        B;                                  /* frames */
    int32_t        width, height;                      /* every image; must equal cam->width / height */
    const uint8_t* img_l;  const uint8_t* img_r;       /* [B][height][width] grey, row-major */
    const int32_t* fast_th;                            /* [B] or NULL; per frame, both images; 0 = ocfg->fast_threshold (:109-111) */
    const int32_t* ll_off; const int32_t* lr_off;      /* [B+1] key lines (octave 0) of the left / right images */
    const float*   seg_l;  const float*   seg_r;       /* [m][4] sPointInOctave{X,Y}, ePointInOctave{X,Y} (= start/end point at octave 0) */
    const float*   angle_l; const float*  angle_r;     /* KeyLine::angle */
    const int32_t* npix_l; const int32_t* npix_r;      /* KeyLine::numOfPixels */
} PlStereoImages;
/* Results and n_stereo equal, byte for byte, what the same inputs give through the three calls
 *   1. plstvo_orb_detect_and_compute_batch on all images, frame f's threshold applied to both of its images;
 *   2. plstvo_lbd_compute_batch on all key lines;
 *   3. plstvo_track_stereo_batch / _sequence on the resulting PlStereoFeatures, with loct_l all 0;
 * but images and key lines go up once and no feature data comes back: ORB's key points and descriptors and LBD's descriptors
 * stay in HBM and feed the stereo step directly.  The host hops after the uploads are ORB's per-image key-point counts (one
 * readback, two under HARRIS_SCORE), the stereo step's survivor counts, and the results.  The sequence form detects and
 * describes each frame's images once.
 * cfg->has_points == 0: ORB does not run (detectStereoPoints returns early in the reference too) and the frames have no key
 * points.  cfg->has_lines == 0: LBD does not run, the frames have no key lines, and every line array may be NULL.
 * fast_th[f] == 0 or fast_th == NULL means ocfg->fast_threshold (detectPointFeatures); values are clamped to [0, 255].  The
 * adaptive threshold of the handler is sequential across frames: a batch or sequence takes the thresholds as given.
 * Returns 0 (a sequence of one frame: 0, no results).  PLSTVO_E_INVALID: a null argument (images where a stage runs), the
 * ORB checks of plstvo_orb_detect_and_compute_batch, or the key-line checks of plstvo_lbd_compute_batch (width / height and
 * numOfPixels 1..32767, offsets that start at 0 and do not decrease); PLSTVO_E_SIZE: prev->B != curr->B, or an image size
 * other than cam's (the reference takes the grid scale from the image, the library from cam); PLSTVO_E_TOO_LARGE: more than
 * PLSTVO_MAX_FEATURES key points or key lines in one image; and the stereo step's matchGrid codes.  The call also updates
 * what plstvo_orb_detect_kernel_times and plstvo_lbd_kernel_times report. */
int plstvo_track_stereo_images_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                     const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlStereoImages* prev,
                                     const PlStereoImages* curr, const PlPrior* priors, PlPoseResult* results,
                                     int32_t* n_stereo /* [B][4], as plstvo_track_stereo_batch */);
int plstvo_track_stereo_images_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                        const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlStereoImages* frames,
                                        const PlPrior* priors, PlPoseResult* results,
                                        int32_t* n_stereo /* [B+1][2], as plstvo_track_stereo_sequence */);

/* ---- stereo images alone in, pose out: the same with LSD inside the call (StereoFrameHandler::initialize / insertStereoPair
 * take images and nothing else, app/imagesStVO.cpp:88-97) ----
 * The signatures of the two calls above plus lcfg.  Results and n_stereo equal, byte for byte, the two-call chain
 *   1. plstvo_lsd_detect_batch(lcfg) on every image, in the images call's block order;
 *   2. plstvo_track_stereo_images_batch / _sequence fed those key lines (angle, numOfPixels, octave 0);
 * and so, through the contract above, LSD -> ORB -> LBD -> plstvo_track_stereo_*.  Each image goes up once and every stage
 * reads that device copy.  With at least as many images in the call as the GPU has SMs, LSD's pixel stages and region growing
 * run on a second stream beside ORB; with fewer, where LSD's one-thread-per-image region growing is the whole critical path and
 * loses more beside ORB than ORB takes, LSD runs first and ORB then runs beside LBD.  What crosses PCIe besides the images and the results is the host hop of the
 * lines: LSD's region counts and records come down, the double cos / sin of the region angles go up, the raw segments come
 * down for the KeyLine step (glibc's atan2f, libstdc++'s std::sort), and the kept key lines go back up with their sincosf
 * direction for LBD; a few KB per image.  The previous images calls' host hops apply as well.
 * The key-line fields of every PlStereoImages (ll_off .. npix_r) must be NULL.  cfg->has_lines == 0: LSD does not run, lcfg
 * may be NULL, and the result is that of the images call without lines; cfg->has_points == 0: ORB does not run.
 * Returns 0 (B == 0, or a sequence of one frame: 0, nothing runs).  PLSTVO_E_INVALID: a non-NULL key-line field, a NULL lcfg
 * with lines on, plstvo_lsd_detect_batch's config checks (refine != 0, scale 0.5, ranges, a blur wider than 31 taps, a scaled
 * size outside 1..32767), more than 65535 images in the call (4 B for a batch, 2 B for a sequence), or a numOfPixels LSD
 * leaves outside 1..32767 (as the chain's step 2 rejects it); PLSTVO_E_TOO_LARGE: more than PLSTVO_MAX_FEATURES key lines in
 * one image (possible with n_features 0); and every code of the images call.  The context stays usable after any error.
 * LSD holds the whole call's images resident: about 35 bytes per scaled pixel (24 MB per 1241x376 image at scale 1.2, so about
 * 12 GB for a 257-frame sequence of 514 images, derived from that figure and not measured) besides the ORB and LBD arenas;
 * PLSTVO_E_CUDA when that cannot be allocated.  The call also updates what plstvo_lsd_kernel_times, plstvo_orb_detect_kernel_times
 * and plstvo_lbd_kernel_times report. */
int plstvo_track_stereo_images_lsd_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                         const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg,
                                         const PlStereoImages* prev, const PlStereoImages* curr, const PlPrior* priors,
                                         PlPoseResult* results, int32_t* n_stereo /* [B][4] */);
int plstvo_track_stereo_images_lsd_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                                            const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                            const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg, const PlStereoImages* frames,
                                            const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo /* [B+1][2] */);

/* Device time of the last images call, ms: [0] image and key-line upload, [1] ORB (pyramid .. descriptors),
 * [2] LBD (gradient + descriptors), [3] stereo step (both passes, all feature sets), [4] f2fTracking + optimizePose.
 * [1] and [2] run on different streams and overlap; a stage that did not run reports 0.  After
 * plstvo_track_stereo_images_lsd_*: [0] ends when LSD starts, and [2] is the lines, from LSD's first launch to LBD's last
 * (to LSD's last where no image has a line), the host hops in between included. */
int plstvo_track_stereo_images_stage_times(PlContext* ctx, float ms5[5]);

/* ---- rectification: what Dataset::nextFrame runs on every frame before the handler (src/dataset.cpp:147-157), i.e.
 * PinholeStereoCamera::rectifyImagesLR (src/pinholeStereoCamera.cpp:188-208): cv::remap(INTER_LINEAR) of each image on the
 * CV_16SC2 maps its constructor built (:30-182) ---- */
typedef struct PlRectifyModel {
    double model;    /* 0: pinhole (cv::initUndistortRectifyMap), 1: equidistant (cv::fisheye::initUndistortRectifyMap) */
    double n_dist;   /* coefficients in D: pinhole 4, 5 or 8 (k1 k2 p1 p2 [k3 [k4 k5 k6]]); fisheye 4 (k1 .. k4) */
    double K[9];     /* camera matrix, row-major (fx, cx, fy, cy are read) */
    double D[8];
    double R[9];     /* rectifying rotation, row-major (cv::stereoRectify's R1 / R2, or the identity) */
    double P[12];    /* new camera matrix, 3x4 row-major; its first three columns are used (stereoRectify's P1 / P2) */
} PlRectifyModel;
/* The CV_16SC2 + CV_16UC1 pair OpenCV 4.13 returns for the model: map1 [height][width][2], map2 [height][width].  Host code,
 * no context or GPU needed; it runs once per rig.  Bit-exact with OpenCV on x86-64 as dispatched for AVX2, whose vector loop
 * sets two things the maps show: the pinhole builder takes each row in blocks of 8 pixels (lane j at the block's start +
 * j * the column step, the leftover columns accumulated), and in those blocks packs the integer coordinate to short with
 * saturation where its scalar loop, the fisheye builder and the leftover columns truncate.  A coordinate * 32 outside int
 * (and the fisheye builder's +-infinity behind the camera) becomes INT_MIN as cvRound gives it.  Exact ties of u * 32 or
 * v * 32, which only rigs with dyadic parameters reach, may round differently where OpenCV's vector code fuses.
 * PLSTVO_E_INVALID: a null pointer, a model other than 0 / 1, a coefficient count other than the above (no thin prism, no
 * tilt), a singular P[:, :3] * R, or width / height outside 1..32767. */
int plstvo_init_undistort_rectify_map(const PlRectifyModel* model, int width, int height, int16_t* map1, uint16_t* map2);

/* A rig's two map pairs resident in HBM, 6 bytes per pixel per side (held once when both sides pass the same pointers, as the
 * reference's cam_d0 branch does).  The maps may come from plstvo_init_undistort_rectify_map or from OpenCV.  Returns NULL on
 * failure (a size outside 1..32767, a null map, or no device memory; plstvo_last_error says which).  Destroy a rectifier
 * before its context. */
typedef struct PlRectifier PlRectifier;
PlRectifier* plstvo_rectifier_create(PlContext* ctx, int width, int height, const int16_t* map1_l, const uint16_t* map2_l,
                                     const int16_t* map1_r, const uint16_t* map2_r);
/* Images of `channels` interleaved 8-bit channels (3: BGR, 4: BGRA, as cv::imread gives them), [height][width][channels]
 * per image.  With maps (all four non-NULL) the device computes cvtColor(remap(img), COLOR_BGR2GRAY) (Dataset::nextFrame's
 * rectifyImagesLR, then the detectors' conversion); with all four NULL, cvtColor alone (the reference's dist == false
 * copy).  The conversion is OpenCV 4.13's for 8-bit data, (3735 B + 19235 G + 9798 R + 2^14) >> 15; alpha is not read.
 * The maps are held as plstvo_rectifier_create holds them.  Every call that takes a rectifier then takes such images in
 * place of grey ones and reads nothing else of them.  Returns NULL on failure; PLSTVO_E_INVALID: channels other than 3 or
 * 4, a size outside 1..32767, some but not all maps NULL (plstvo_last_error says which). */
PlRectifier* plstvo_rectifier_create_color(PlContext* ctx, int width, int height, int channels,
                                           const int16_t* map1_l, const uint16_t* map2_l,
                                           const int16_t* map1_r, const uint16_t* map2_r);
void plstvo_rectifier_destroy(PlRectifier* rect);
/* rectifyImagesLR on B pairs: out_l[b] = cv::remap(img_l[b], map1_l, map2_l, INTER_LINEAR, BORDER_CONSTANT, 0), and the
 * same on the right; images [B][height][width][channels] of the rectifier's size and channels in, [B][height][width] grey
 * out, host memory.  The weights are OpenCV's INTER_LINEAR table and the sum is rounded as cv::remap rounds it, so the result
 * equals OpenCV's byte for byte.  A colour rectifier converts each remapped image (or, without maps, each image) with
 * cvtColor(COLOR_BGR2GRAY), byte for byte too.  PLSTVO_E_INVALID: a null pointer, B < 0, or a rectifier of another context.
 * Device memory: channels + 1 bytes per pixel of the call (raw and grey), kept by the context for the next call. */
int plstvo_rectify_batch(PlContext* ctx, const PlRectifier* rect, int B, const uint8_t* img_l, const uint8_t* img_r,
                         uint8_t* out_l, uint8_t* out_r);
/* Device time of the last remap or colour preparation on this context (plstvo_rectify_batch or a raw-images call), ms. */
int plstvo_rectify_kernel_times(PlContext* ctx, float* ms1);

/* ---- raw stereo images in, pose out: Dataset::nextFrame's rectifyImagesLR, then the handler (plstvo_track_stereo_images_lsd_*)
 * The signatures of the _lsd_ calls plus rect.  Results and n_stereo equal, byte for byte, plstvo_rectify_batch on every pair
 * followed by plstvo_track_stereo_images_lsd_batch / _sequence on the rectified images.  rect == NULL: the _lsd_ call (the
 * reference's copy when dist is false).  PlStereoImages' img_l / img_r are [B][height][width][channels] of the rectifier
 * (colour images for a colour rectifier).  The raw images go up once into a staging slot and the remap (for colour images,
 * the remap and the conversion to grey, or the conversion alone) writes the grey device copy that LSD, ORB and LBD read, so
 * no rectified image crosses PCIe and no stage reads the caller's images; stage slot [0] of
 * plstvo_track_stereo_images_stage_times then covers the upload and the remap.  Device memory besides the _lsd_ call's: the
 * staging copy, channels bytes per pixel of the call, and the rectifier's maps.  PLSTVO_E_SIZE: the rectifier's size differs
 * from cam's (and so from the images');
 * PLSTVO_E_INVALID: a rectifier of another context, and every code of the _lsd_ calls.  The context stays usable after any
 * error.  The call also updates what plstvo_rectify_kernel_times reports when the images are read. */
int plstvo_track_stereo_raw_images_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                         const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg,
                                         const PlRectifier* rect, const PlStereoImages* prev, const PlStereoImages* curr,
                                         const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo /* [B][4] */);
int plstvo_track_stereo_raw_images_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                                            const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                            const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg, const PlRectifier* rect,
                                            const PlStereoImages* frames, const PlPrior* priors, PlPoseResult* results,
                                            int32_t* n_stereo /* [B+1][2] */);

/* ---- stereo sessions: StereoFrameHandler's prev_frame kept on the device for many independent streams
 * (app/imagesStVO.cpp:88-124, src/stereoFrameHandler.cpp:35-102) ----
 * A session holds, for each of n_streams independent stereo streams (cameras), the previous frame's stereo features in HBM,
 * as the tracker reads them in the previous-frame role: per kept stereo point 64 bytes (P 24, sigma2 8, descriptor 32), per
 * kept stereo line 124 bytes (start / end points 16 + 16, sP / eP 24 + 24, sigma2 8, level 4, descriptor 32).  The session
 * has two such pools (the kept frames, and the next call's), each grown on demand with a quarter of slack; it keeps no
 * images, on the host or the device.  Features carry no state from one frame to the next in the reference (matchF2FPoints /
 * matchF2FLines flag copies, updateFrame moves curr_frame into prev_frame), so a frame's stereo features are computed once
 * and serve as the next pair's previous frame unchanged.
 * The configs are copied at creation and fixed for the session's life (the kept records depend on cam and scfg, the
 * descriptors on ocfg and lcfg).  lcfg may be NULL where cfg->has_lines is 0.  rect (NULL: the images are already rectified)
 * must belong to ctx and outlive the session; the frames of _initialize / _insert are [height][width][channels] of it, so a
 * colour rectifier takes colour frames.  Returns NULL on failure (a null argument, n_streams < 1, the ORB / LSD config
 * checks of the _lsd_ calls, a bad grid, a rectifier of another context or of another size; plstvo_last_error says which).
 * Destroy a session before its context; plstvo_stereo_session_device_bytes is its device memory (pools and call tables). */
typedef struct PlStereoSession PlStereoSession;
PlStereoSession* plstvo_stereo_session_create(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                                              const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                              const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg, const PlRectifier* rect,
                                              int n_streams);
/* A session whose stream i is tracked under its own camera cams[i] and prepared by its own rectifier rects[i]: N
 * StereoFrameHandlers, each built on its own PinholeStereoCamera (app/imagesStVO.cpp:66,86, src/stereoFrameHandler.cpp:29).
 * Every camera must have one width / height (PLSTVO_E_SIZE otherwise); the configs are those of plstvo_stereo_session_create.
 * rects == NULL (or every entry NULL): no stream is remapped.  In a grey session rects[i] == NULL takes stream i's images as
 * given.  Every non-NULL rectifier must belong to ctx (PLSTVO_E_INVALID) and have the cameras' size (PLSTVO_E_SIZE), and all
 * must have one channel count (PLSTVO_E_INVALID).  A colour session needs a colour rectifier for every stream
 * (PLSTVO_E_INVALID for a NULL entry): give one without maps where a camera needs no remap.  Rectifiers must outlive the
 * session.  _initialize, _insert, _retain, _read, _device_bytes and _destroy work on it unchanged.
 * Contract: without rectifiers, each stream's results, n_stereo and _read rows equal, byte for byte, those of a
 * plstvo_stereo_session_create session with that stream's camera driven through the same calls; with rectifiers, those of
 * the same session without them fed each stream's frames after plstvo_rectify_batch with its rectifier.  Device memory
 * besides the plain session's: a call table of n cameras (48 bytes each, counted by plstvo_stereo_session_device_bytes) and,
 * with rectifiers, a table of 2 n map pointers beside the call's staged images. */
PlStereoSession* plstvo_stereo_session_create_cams(PlContext* ctx, const PlCamera* cams /* [n_streams] */, const PlConfig* cfg,
                                                   const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                                   const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg,
                                                   const PlRectifier* const* rects /* [n_streams] or NULL */, int n_streams);
void    plstvo_stereo_session_destroy(PlStereoSession* s);
int64_t plstvo_stereo_session_device_bytes(const PlStereoSession* s);
/* StereoFrameHandler::initialize(img_l, img_r) for streams ids[0 .. n) (any subset of [0, n_streams), any order, no
 * duplicates): frames (B = n, the _lsd_ calls' frames: key-line fields NULL) are detected, go through the stereo step and
 * replace each named stream's kept frame.  frames->fast_th[k] is stream ids[k]'s FAST threshold for its frame (0 or NULL:
 * ocfg->fast_threshold).  n_stereo [n][2] (optional): each new frame's stereo points, lines. */
int plstvo_stereo_session_initialize(PlContext* ctx, PlStereoSession* s, int n, const int32_t* ids,
                                     const PlStereoImages* frames, int32_t* n_stereo);
/* insertStereoPair's f2fTracking + optimizePose for streams ids[0 .. n), each of which must hold a frame: the new frame k is
 * tracked against stream ids[k]'s kept frame and then replaces it; streams not named keep their frame untouched.  results and
 * n_stereo ([n][4]: the kept frame's stereo points, lines, then the new frame's) equal, byte for byte, those of
 * plstvo_track_stereo_raw_images_batch with the session's rect and configs, prev = each named stream's kept images at the
 * threshold they were detected with, curr = frames, the same priors ([n] or NULL) and the same order (rect NULL:
 * plstvo_track_stereo_images_lsd_batch).  Only the 2 n new images are uploaded, rectified, detected and described, and only
 * the new frames go through the stereo step; the kept frames are gathered on the device (session_gather_kernel).
 * Both calls return 0 or an error code, and a failed call leaves every stream's kept frame as it was and the context usable.
 * PLSTVO_E_INVALID: a null session, a session of another context, ids null, an id outside [0, n_streams), a duplicate id,
 * insert on a stream with no frame, more than 65535 images in the call (2 n), and every PLSTVO_E_INVALID of the _lsd_ /
 * raw-images calls; PLSTVO_E_SIZE: frames->B != n, and that call's size codes; PLSTVO_E_TOO_LARGE: its feature limits, or
 * more than INT_MAX kept rows; PLSTVO_E_CUDA: among others, when a pool cannot be grown.  insert updates what
 * plstvo_track_stereo_images_stage_times and the ORB / LSD / LBD / rectify kernel-time calls report, as the images calls do
 * (initialize too, its tracking slot then empty). */
int plstvo_stereo_session_insert(PlContext* ctx, PlStereoSession* s, int n, const int32_t* ids, const PlStereoImages* frames,
                                 const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo);
/* The reference's FLD line branch (use_fld_lines, src/stereoFrame.cpp:244-304) on a session: on != 0 makes _initialize,
 * _insert, _run and _run_keyframes take each frame's key lines from the caller instead of running LSD, off (the state at
 * creation) restores LSD.  Legal only while no stream holds a frame (PLSTVO_E_INVALID otherwise, the session unchanged), so
 * every kept frame of a session was described one way; it works on _create and _create_cams sessions alike, and lcfg,
 * checked at creation as before, is not read while it is on.
 * With it on, wherever cfg->has_lines is set the frames' key-line fields (ll_off .. npix_r) are required and hold what the
 * images call takes (plstvo_fld_key_lines' rows: sPointInOctave / ePointInOctave, angle, numOfPixels), frame-major for
 * _initialize / _insert and step-major over the T n frames of a run, with plstvo_lbd_compute_batch's key-line checks
 * (PLSTVO_E_INVALID for a missing or malformed field or a numOfPixels outside 1..32767; PLSTVO_E_TOO_LARGE for more than
 * PLSTVO_MAX_FEATURES lines in one image); where has_lines is 0 they must be NULL (PLSTVO_E_INVALID).  Each such error
 * leaves the session usable.  LSD does not run and LBD describes the given lines; a run describes all 2 n T images' lines in
 * one LBD pass and keeps no LSD arena.  Contract: an insert equals plstvo_track_stereo_images_batch with the session's
 * configs, prev = each named stream's kept images and key lines at their thresholds, curr = frames, the same priors; the
 * runs equal T such inserts as plstvo_stereo_session_run states it.  Retention, _read, _read_keyframes (ls_src: the row
 * in the caller's key lines of the image) work unchanged.
 * A colour session computes the branch's fld_img = cvtColor(img, CV_RGB2GRAY) of each remapped (or unmapped) image beside
 * the COLOR_BGR2GRAY copy ORB reads, in the same launch, and LBD reads it: one byte per pixel of the call more of the
 * rectifier's staging. */
int plstvo_stereo_session_use_fld_lines(PlContext* ctx, PlStereoSession* s, int on);

/* ---- reading a session call's frames back: StereoFrame::stereo_pt / stereo_ls and StereoFrameHandler::matched_pt / _ls
 * of the last _initialize / _insert ----
 * Outputs of plstvo_stereo_session_read.  Every pointer may be NULL (that array is not copied).  The point and line fields
 * are what plstvo_match_stereo_points / _lines write for the call's n new frames, in call order, frame k's rows after frame
 * k - 1's; the row counts are the call's n_stereo (initialize: columns 0, 1; insert: columns 2, 3).  pt_src / ls_src are
 * their src_idx: the index in ORB's / LSD's output order for the left image.  m12_* and inlier_* (insert only) are what
 * plstvo_track_batch writes, one row per feature of each named stream's kept (previous) frame in call order (the insert's
 * n_stereo columns 0, 1), an m12 value indexing the stream's new frame's rows (or -1). */
typedef struct PlStereoFrameOut {
    double* pt_pl; double* pt_disp; double* pt_P; double* pt_sigma2; int32_t* pt_level; uint8_t* pdesc; int32_t* pt_src;
    double* ls_spl; double* ls_epl; double* ls_sdisp; double* ls_edisp; double* ls_sP; double* ls_eP; double* ls_le;
    double* ls_angle; double* ls_sigma2; int32_t* ls_level; uint8_t* ldesc; int32_t* ls_src;
    int32_t* m12_pt; uint8_t* inlier_pt; int32_t* m12_ls; uint8_t* inlier_ls;
} PlStereoFrameOut;
/* Retention switch, off at creation.  on != 0 takes effect from the next _initialize / _insert: each successful call then
 * keeps, in a session-owned device arena (counted by plstvo_stereo_session_device_bytes, untouched by other calls on the
 * context), its new frames' full records (96 bytes per stereo point, 176 per stereo line) and, for an insert, the tracker's
 * m12 and inlier rows (5 bytes per kept row).  Filling it costs two more lift launches per call and device-to-device copies.
 * on == 0 frees the arena at once; with retention off a call's launches, device memory and results are those of a session
 * never switched on.  Returns 0, or PLSTVO_E_INVALID for a null or foreign session. */
int plstvo_stereo_session_retain(PlContext* ctx, PlStereoSession* s, int on);
/* Copies what the last call retained into out's non-NULL arrays (after an initialize, m12_* and inlier_* are left untouched)
 * and returns that call's n.  PLSTVO_E_INVALID: ctx, s or out null, a session of another context, retention off, no call
 * succeeded since retention was turned on, or the last call on the session failed (any failed call discards what was
 * retained, so a read never mixes two calls). */
int plstvo_stereo_session_read(PlContext* ctx, const PlStereoSession* s, const PlStereoFrameOut* out);
/* ---- drawing each new frame: StereoFrame::plotStereoFrame (src/stereoFrame.cpp:618-663), the image app/imagesStVO.cpp:109
 * hands its scene ----
 * Plot switch, off at creation.  on != 0 requires retention on (PLSTVO_E_INVALID otherwise) and takes effect from the next
 * _initialize / _insert: each successful call then also draws, for each new frame in call order, the image the reference's
 * curr_frame->plotStereoFrame() returns for it: the frame's left image after the session's rectification (its stream's
 * rectifier on a _create_cams session) in BGR (a grey image replicated, as cvtColor(GRAY2BGR); BGRA with alpha dropped, as
 * cvtColor(BGRA2BGR)), then cv::circle(img, Point(int(pl.x), int(pl.y)), 3, Scalar(0, 200, 0), 1) for every row of pt_pl
 * and cv::line(img, Point(int(spl.x), int(spl.y)), Point(int(epl.x), int(epl.y)), Scalar(0, 200, 0), 1) for every row of
 * ls_spl / ls_epl that plstvo_stereo_session_read returns for the call, both LINE_8, byte for byte with OpenCV 4.13 (clipped
 * at the border, each line drawn from spl to epl).  It costs one base-image launch and, where the call has a point or a line,
 * one drawing launch per call, and a session-owned arena of 3 bytes per pixel per new frame (counted by
 * plstvo_stereo_session_device_bytes), plus 16 bytes per new frame for a colour session's map table and, where no stage of
 * the call reads the images on the device (a grey session without a rectifier and with has_points 0), 1 byte per pixel per
 * new frame for their upload.  With plotting on the call's frames must hold both images (PLSTVO_E_INVALID otherwise), even
 * where has_points and has_lines are 0.  on == 0 frees the arena at once, as does retention off, which also turns plotting
 * off; with plotting off a call's launches, device memory and results are those of a session never switched on, and with
 * it on its results, n_stereo and _read rows are the same.  _run, _run_keyframes and _run_schedule draw nothing.  Returns
 * 0, or PLSTVO_E_INVALID for a null or foreign session or retention off. */
int plstvo_stereo_session_plot(PlContext* ctx, PlStereoSession* s, int on);
/* Copies the last call's images, [n][height][width][3] BGR bytes in call order, into out and returns that call's n.
 * PLSTVO_E_INVALID: ctx, s or out null, a session of another context, plotting off, no _initialize / _insert succeeded
 * since plotting was turned on, the last call on the session failed, or it was a run (every run, even of T = 0, discards the
 * last plot, as any failed call does). */
int plstvo_stereo_session_read_plot(PlContext* ctx, const PlStereoSession* s, uint8_t* out /* [n][height][width][3] */);

/* ---- running the handler's frame loop over many frames per stream in one call (app/imagesStVO.cpp:88-124) ----
 * The Config values of updateFrame's adaptive FAST threshold (include/config.h:50, :67-71; src/config.cpp:52, :72-76).
 * fast_err_th is a float, as updateFrame reads it (src/stereoFrameHandler.cpp:72). */
typedef struct PlHandlerConfig {
    int32_t adaptative_fast;
    int32_t fast_min_th, fast_max_th, fast_inc_th, fast_feat_th;
    float   fast_err_th;
} PlHandlerConfig;
void plstvo_default_handler_config(PlHandlerConfig* h);   /* 1, 5, 50, 5, 50, 0.5f (src/config.cpp) */
void plstvo_kitti_handler_config(PlHandlerConfig* h);     /* 1, 7, 30, 5, 50, 0.5f (config/config/config_kitti.yaml) */
/* T steps of StereoFrameHandler's loop (insertStereoPair, optimizePose, updateFrame) for streams ids[0 .. n), each of which
 * must hold a frame.  frames holds B = T * n frames, step-major: frame t * n + k is stream ids[k]'s frame of step t; its
 * fast_th and key-line fields must be NULL.  Contract: the call equals, byte for byte, T calls of
 * plstvo_stereo_session_insert on the same session, where the call of step t takes step t's n frames with
 *   thresholds th_t:  th_0[k] = fast_th0[k] (fast_th0 NULL or an entry 0: ocfg->fast_threshold, as the images calls map it);
 *                     th_{t+1}[k] = updateFastThreshold(h, th_t[k], curr_frame, results[t][k].n_inliers_pt) (plstvo.hpp);
 *   priors:           priors at t = 0 (NULL as for insert), then priorOf of the frame publishPose(results[t - 1][k]) fills.
 * Under it, results ([T][n]), n_stereo ([T][n][4], optional), the threshold rows (fast_th [T + 1][n], optional: row t = th_t,
 * row T the threshold the next frame would take), the kept frames (a further insert gives the same bytes) and, with
 * retention on, what plstvo_stereo_session_read returns (the last step, as if it had been an insert) are equal.  Streams not
 * named are untouched.  T = 0 returns 0 and changes nothing; fast_th's row 0 (= row T) is still written.  A second run
 * continues a first exactly when given fast_th0 = row T and priors built from the last results, so the caller splits a long
 * sequence into calls of the T that fits.
 * Schedule: all 2 n T images go up once and are rectified / converted once; LSD and LBD run once over all of them; then each
 * step runs ORB at the device threshold row, the stereo step, tracking, and session_handler_kernel, which writes the next
 * threshold row and the next priors on the device.  Per step, the host hops are an insert's: ORB's key-point counts and the
 * stereo step's survivor counts.  The results, n_stereo rows and thresholds come down once, at the end.
 * Device memory besides the session's pools: every image of the call is resident at once: LSD's 35 bytes or so per scaled
 * pixel (as the _lsd_ calls), the grey copy's 1 byte per pixel, and with a rectifier its staging copy's channels bytes per
 * pixel; LBD's outputs for all the call's key lines; and a table of T n results and 2 (T + 1) n thresholds.  The caller picks
 * T to fit.  plstvo_track_stereo_images_stage_times then covers the whole call: [0] uploads and preparation, [1] ORB summed
 * over the steps, [2] LSD + LBD, [3] the stereo step summed, [4] tracking and the threshold / prior update summed; the
 * kernel-time calls report their last launches.
 * Checks before any work, each leaving the session and context usable: PLSTVO_E_INVALID for h NULL; h out of range
 * (fast_min_th < 1, fast_min_th > fast_max_th, fast_max_th > 255, fast_inc_th < 0, fast_feat_th < 0, a non-finite
 * fast_err_th; the floor of 1 keeps a threshold of 0 from meaning the configured one); a non-NULL frames->fast_th or key-line
 * field; a fast_th0 entry, or an ocfg->fast_threshold it maps to, outside [0, 255] (the rule sees what ORB uses); T < 0; more
 * than 65535 images (2 n T); a session whose ocfg.n_features exceeds PLSTVO_MAX_FEATURES (so no step can fail on a feature
 * limit); and insert's id, liveness and config checks.  PLSTVO_E_SIZE: frames->B != T * n, and insert's size codes.
 * LSD's key-line limit (PLSTVO_E_TOO_LARGE) is found before step 0, since LSD runs first.
 * Not checked before any work: the limits the T inserts would meet step by step (matchGrid's 128 candidates in one query
 * window, the per-pair solver's list capacity, more than INT_MAX kept rows) and CUDA failures.  Such an error part-way
 * returns its code with the named streams holding the frames of the last completed step, but results, fast_th and
 * n_stereo are then unspecified and the number of completed steps is not returned, so the caller cannot continue exactly
 * from there: it re-initialises those streams and continues with per-frame inserts or a new run.  For a CUDA failure this
 * is not verified, since nothing provokes one safely. */
int plstvo_stereo_session_run(PlContext* ctx, PlStereoSession* s, const PlHandlerConfig* h, int n, const int32_t* ids, int T,
                              const PlStereoImages* frames, const int32_t* fast_th0 /* [n] or NULL */,
                              const PlPrior* priors /* [n] or NULL */, PlPoseResult* results /* [T][n] */,
                              int32_t* fast_th /* [T + 1][n] or NULL */, int32_t* n_stereo /* [T][n][4] or NULL */);

/* ---- the same loop with the PL-SLAM key-frame test (needNewKF / currFrameIsKF, src/stereoFrameHandler.cpp:1136-1218) ----
 * The Config values of needNewKF (include/config.h:39-41, :108-110; defaults src/config.cpp:40-42).  -inf / +inf switch a
 * criterion off; NaN is refused. */
typedef struct PlKeyframeConfig {
    double min_entropy_ratio, max_kf_t_dist, max_kf_r_dist;
} PlKeyframeConfig;
void plstvo_default_keyframe_config(PlKeyframeConfig* k);   /* 0.85, 5.0, 15.0 */
/* One stream's key-frame state, the handler's SLAM variables (include/stereoFrameHandler.h:81-86), as plstvo.hpp's
 * KeyframeTest holds them.  T_prevKF and cov_prevKF_currF are row-major. */
typedef struct PlKeyframeState {
    int32_t prev_f_iskf, N_prevKF_currF;
    double  entropy_first_prevKF;
    double  T_prevKF[16];
    double  cov_prevKF_currF[36];
} PlKeyframeState;
void plstvo_initial_keyframe_state(PlKeyframeState* s);     /* what initialize() leaves (:48-51): 1, 0, 0.0, I, 0 */
/* One stream's needNewKF at one step: the decision, N_prevKF_currF as needNewKF leaves it (before currFrameIsKF resets it),
 * and the test's entropy of the accumulated covariance, its ratio to the key frame's, and the distance t (m) and angle r
 * (degrees) to the previous key frame. */
typedef struct PlKeyframeResult {
    int32_t new_kf, N_prevKF_currF;
    double  entropy_curr, entropy_ratio, t, r;
} PlKeyframeResult;
/* plstvo_stereo_session_run with, per named stream and step, needNewKF after optimizePose and currFrameIsKF where it fires,
 * before updateFrame.  Contract: the call equals T calls of plstvo_stereo_session_insert on the same session as the run's
 * contract states them, except that the prior of step t + 1 is priorOf of the published frame with Tfw = I and Tfw_cov = I
 * where kf[t][k].new_kf is 1, and that each step's results go through plstvo.hpp's KeyframeTest::needNewKF, starting from
 * kf_state[k].  Under it results (optimizePose's rows, Tfw before any reset), n_stereo and fast_th are byte for byte the
 * loop's; kf[t][k].new_kf and .N_prevKF_currF are the host test's; the four diagnostics agree with it to the last few ulps
 * (the device's log and acos are CUDA's); and kf_state comes back as the host test stands after step T - 1.  The decisions
 * are held to the reference's own needNewKF, not only to the host test: wherever t, r and the entropy ratio lie outside the
 * rounding band of their thresholds they are the exact ones, and on non-finite poses and covariances (a NaN cosine keeps
 * r = 0; a zero pivot with inf or NaN below it gives a NaN determinant) they are the reference's.  Inside a band (a few ulps
 * of fp64's log, acos and summation order) either decision may be taken.
 * A second call continues a first exactly when given fast_th0 = row T, the returned kf_state, and priors built from the last
 * results with that reset applied.
 * The test runs in session_keyframe_kernel, one thread per stream after session_handler_kernel: one launch per step more
 * than plstvo_stereo_session_run, in fp64 without fused multiply-adds.
 * Retention (plstvo_stereo_session_retain on): the call keeps, for every (step, stream) whose frame became a key frame,
 * that frame's new stereo points and lines, the same bytes as an insert of that frame retains; plstvo_stereo_session_read
 * still returns the last step.  The device arena grows by each step's new rows of every named stream, 96 bytes per stereo
 * point and 176 per stereo line, in one allocation per step with the session's usual slack (a quarter more, plus 256-byte
 * alignment per array; counted by plstvo_stereo_session_device_bytes), and every step is retained as an insert
 * is, so a retained call costs two lift launches, the tracker's row copies and one copy launch more per step.
 * Checks before any work: those of plstvo_stereo_session_run, and PLSTVO_E_INVALID for k, kf_state or kf NULL, a NaN in k,
 * and a kf_state entry with prev_f_iskf outside {0, 1} or N_prevKF_currF < 0.  A failed call leaves kf_state untouched and
 * discards the key frames (as it discards what _read returns); so does any other call on the session. */
int plstvo_stereo_session_run_keyframes(PlContext* ctx, PlStereoSession* s, const PlHandlerConfig* h, const PlKeyframeConfig* k,
                                        int n, const int32_t* ids, int T, const PlStereoImages* frames,
                                        const int32_t* fast_th0 /* [n] or NULL */, const PlPrior* priors /* [n] or NULL */,
                                        PlKeyframeState* kf_state /* [n] in / out */, PlPoseResult* results /* [T][n] */,
                                        PlKeyframeResult* kf /* [T][n] */, int32_t* fast_th /* [T + 1][n] or NULL */,
                                        int32_t* n_stereo /* [T][n][4] or NULL */);
/* ---- the frame loop over uneven streams: a per-step, per-stream schedule (app/imagesStVO.cpp:88-124 per camera) ----
 * _run and _run_keyframes where a stream may have no frame at a step, start inside the call, or be re-initialised:
 * schedule [T][n] holds, for stream ids[k] at step t,
 *   0  no frame: the stream idles, its kept frame, threshold, prior and key-frame state carried unchanged;
 *   1  insert: insertStereoPair + optimizePose (+ needNewKF / currFrameIsKF with k) + updateFrame, as _run's step;
 *   2  initialize: StereoFrameHandler::initialize on this frame (src/stereoFrameHandler.cpp:35-52).
 * frames holds B = the number of non-zero entries, step-major and within a step in ids order (FLD sessions: the key-line
 * fields in the same order).  frames->fast_th is NULL or [B]: an initialize entry's threshold as _initialize takes it (0:
 * ocfg->fast_threshold, Config::orbFastTh as HandlerState's initialize starts from), and 0 for every insert entry.
 * k == NULL: no key-frame test, and kf_state and kf must be NULL; else the test of _run_keyframes, kf_state [n] in / out.
 * Contract: the call equals, byte for byte, this chain on the same session.  For t = 0 .. T - 1, one
 * plstvo_stereo_session_initialize on step t's code-2 entries (in ids order, at their thresholds), then one
 * plstvo_stereo_session_insert on its code-1 entries; a chain call with no entries is not made.  Per stream, the insert
 * takes the threshold and prior _run / _run_keyframes would carry to it (th_0 = fast_th0 as _run maps it, priors [n] or
 * NULL at the call's start), and the key-frame state from kf_state; an idle step carries all three unchanged; an
 * initialize resets them to what HandlerState's initialize leaves: the entry's threshold, priorOf of the fresh frame (Tfw = I,
 * Tfw_cov = I, DT = I, DT_cov = 0, err_norm = -1) and plstvo_initial_keyframe_state.  priors NULL starts every stream from
 * that fresh prior too, which optimizePose treats as insert's NULL (err_norm < 0 fails isGoodSolution).
 * Under it: results [T][n] and kf [T][n] are written for code-1 entries only (other rows untouched); n_stereo [T][n][4]
 * is insert's row for a code-1 entry and {0, 0, points, lines} for a code-2 entry (idle rows untouched); fast_th [T + 1][n]
 * row t holds the threshold each stream's frame of step t was detected with, and for an idle stream its carried threshold
 * (the one its next insert would take); row T the carried thresholds after the call, as in _run; kf_state comes back as the chain's test stands after step T - 1; the
 * kept frames, what plstvo_stereo_session_read returns (the last step with any entry, as its last chain call retains it:
 * the insert when the step has both kinds) and with k what plstvo_stereo_session_read_keyframes returns (rows' step is the
 * step t) are the chain's.  Every entry 1 is the existing run: the outputs equal _run (k NULL) and _run_keyframes (k set).
 * T = 0, or no non-zero entry, runs nothing: fast_th's rows are all row 0 and what _read returns is left as _run leaves it
 * (k set: no key frames kept, as _run_keyframes).  A second call continues a first exactly as _run_keyframes states it.
 * Work: the 2 B present images go up once and are rectified / converted per group (each group's streams' rectifiers) into
 * one device copy; LSD (or the FLD cut of the caller's lines) and LBD run once over all of them, one line block per image.
 * Then each step with entries runs its initialize group (ORB at the host thresholds, the stereo step, the session's
 * commit), then its insert group (ORB at thresholds gathered on the device, the stereo step, tracking and the handler update),
 * each group as _initialize / _insert would, so a step with both kinds costs two groups' host hops (ORB's key-point counts,
 * the stereo step's survivor counts, and the initialize group's final synchronise) instead of one.  A step with no entries
 * costs nothing.  The threshold, prior and key-frame state of each named stream stay in a device slot for the whole call:
 * session_schedule_gather_kernel reads an insert group's from the slots before its ORB, and session_schedule_update_kernel
 * writes them back after its test (or resets an initialize group's); idle slots are not touched.  Moves and integer
 * writes only; the arithmetic stays in session_handler_kernel and session_keyframe_kernel.
 * Device memory besides the session's pools: _run's, with B present frames for T n, plus the slots (n thresholds, priors
 * and key-frame states), a [T + 1][n] threshold table and the largest insert group's threshold rows and states.  With a
 * rectifier each group's images pass the rectifier's staging, then are copied into the call's grey copy (twice with the
 * colour FLD branch's RGB2GRAY plane).  plstvo_track_stereo_images_stage_times then covers the whole call as for _run: [0]
 * uploads and preparation, [1] ORB summed over the groups, [2] LSD + LBD, [3] the stereo step summed, [4] tracking and the
 * state updates summed.
 * Checks before any work, each leaving the session and context usable: every check of _run (k NULL) or _run_keyframes (k
 * set), with the image limit counting the present images only (2 B > 65535), plus PLSTVO_E_INVALID for a schedule value
 * outside {0, 1, 2}, a NULL schedule with T n > 0, kf_state or kf non-NULL with k NULL, a code-1 entry for a stream that
 * holds no frame at that step (it held one at the call's start or had an earlier code-2 entry in the call), a non-zero
 * frames->fast_th of a code-1 entry and an initialize threshold outside [0, 255]; PLSTVO_E_SIZE for frames->B != the
 * number of non-zero entries.  A failure part-way follows _run's rule. */
int plstvo_stereo_session_run_schedule(PlContext* ctx, PlStereoSession* s, const PlHandlerConfig* h, const PlKeyframeConfig* k,
                                       int n, const int32_t* ids, int T, const uint8_t* schedule /* [T][n] */,
                                       const PlStereoImages* frames, const int32_t* fast_th0 /* [n] or NULL */,
                                       const PlPrior* priors /* [n] or NULL */, PlKeyframeState* kf_state /* [n] or NULL */,
                                       PlPoseResult* results /* [T][n] */, PlKeyframeResult* kf /* [T][n] or NULL */,
                                       int32_t* fast_th /* [T + 1][n] or NULL */, int32_t* n_stereo /* [T][n][4] or NULL */);
/* Copies the key frames the last plstvo_stereo_session_run_keyframes kept into out's non-NULL point and line arrays, in
 * (step, call position) order, key frame j's rows after key frame j - 1's (m12_* / inlier_* are not read), and writes
 * rows [n_kf][4]: step, stream id, stereo points, stereo lines (rows may be NULL to learn n_kf).  Returns n_kf.
 * PLSTVO_E_INVALID: ctx, s or out null, a session of another context, retention off, or no key frames kept (the last call
 * on the session was not a successful run_keyframes). */
int plstvo_stereo_session_read_keyframes(PlContext* ctx, const PlStereoSession* s, const PlStereoFrameOut* out,
                                         int32_t* rows /* [n_kf][4] or NULL */);

/* ---- include/stereoFrameHandler.h surface ----------------------------------------------------- */
/* StereoFrameHandler::f2fTracking (src/stereoFrameHandler.cpp:106-180) for B independent
 * (prev, curr) pairs: descriptor matching for points and lines; m12_* hold problem-local indices
 * (prev row -> curr row or -1).  n_matched[2*p], [2*p+1] = matched_pt.size(), matched_ls.size(). */
int plstvo_f2f_tracking(PlContext* ctx, const PlConfig* cfg, const PlFrameBatch* prev,
                        const PlFrameBatch* curr, int32_t* m12_pt, int32_t* m12_ls, int32_t* n_matched);

/* StereoFrameHandler::optimizePose (src/stereoFrameHandler.cpp:307-392) on explicit matched lists.
 * priors may be NULL (identity Tfw, no motion-model state).  inlier_* (optional) receive the
 * final PointFeature::inlier / LineFeature::inlier flags in list order. */
int plstvo_optimize_pose(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                         const PlMatchedBatch* matched, const PlPrior* priors,
                         PlPoseResult* results, uint8_t* inlier_pt, uint8_t* inlier_ls);

/* insertStereoPair's f2fTracking + optimizePose (app/imagesStVO.cpp:96-97) for B independent pairs,
 * entirely on the device: match -> build matched_pt/ls (ascending prev index, with the
 * LineFeature::safeCopy sigma2 rule) -> optimizePose.  Host buffers in, host buffers out;
 * H2D / compute / D2H are pipelined over chunks of pairs.
 * m12_* / inlier_* are indexed by prev-frame feature (problem-local curr index or -1; 1 = matched and
 * still an inlier after optimizePose).  Any output pointer may be NULL. */
int plstvo_track_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                       const PlFrameBatch* prev, const PlFrameBatch* curr, const PlPrior* priors,
                       PlPoseResult* results, int32_t* m12_pt, int32_t* m12_ls,
                       uint8_t* inlier_pt, uint8_t* inlier_ls);

/* plstvo_track_batch with pair p solved under cams[p] (B cameras: several calibrated rigs in one batch).  Row p of every
 * output equals row p of plstvo_track_batch on the same inputs with cam = cams[p], byte for byte: matching does not read the
 * camera, the solver plan depends on B and the list lengths only, and each pair is solved on its own.  Same H2D / compute /
 * D2H pipeline and errors as plstvo_track_batch (PLSTVO_E_INVALID for cams NULL); device memory besides its: B x 48 bytes. */
int plstvo_track_batch_cams(PlContext* ctx, const PlCamera* cams /* [B] */, const PlConfig* cfg,
                            const PlFrameBatch* prev, const PlFrameBatch* curr, const PlPrior* priors,
                            PlPoseResult* results, int32_t* m12_pt, int32_t* m12_ls,
                            uint8_t* inlier_pt, uint8_t* inlier_ls);

/* Streaming form of plstvo_track_batch: enqueues the batch (H2D, kernels, D2H) and returns a ticket >= 0 without
 * waiting, so that the caller can submit batch k+1 (its H2D then overlaps the kernels of batch k) before it waits for
 * batch k.  Two batches may be in flight per context; all input AND output buffers of a batch must stay valid and
 * untouched until plstvo_wait(ticket) returned (use plstvo_host_alloc memory: pageable memory makes the copies
 * synchronous).  This is how a video pipeline drives the engine: frame k+1's features go up while pair k solves. */
int plstvo_track_batch_async(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                             const PlFrameBatch* prev, const PlFrameBatch* curr, const PlPrior* priors,
                             PlPoseResult* results, int32_t* m12_pt, int32_t* m12_ls,
                             uint8_t* inlier_pt, uint8_t* inlier_ls);
int plstvo_wait(PlContext* ctx, int ticket);

/* ---- throughput mode: inputs resident in HBM -------------------------------------------------- */
int  plstvo_batch_upload(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                         const PlFrameBatch* prev, const PlFrameBatch* curr, const PlPrior* priors,
                         PlDeviceBatch** out);
/* one pass of the hot path over the resident batch (no host<->device traffic); asynchronous */
int  plstvo_batch_run(PlContext* ctx, PlDeviceBatch* db);
/* run `iters` passes bracketed by CUDA events on the launching stream; *ms_total = elapsed.
 * flush_l2 != 0 writes a buffer larger than L2 between passes (outside the per-pass events, so
 * ms_total only sums the passes). */
int  plstvo_batch_run_timed(PlContext* ctx, PlDeviceBatch* db, int iters, int flush_l2, float* ms_total);
int  plstvo_batch_download(PlContext* ctx, PlDeviceBatch* db, PlPoseResult* results,
                           int32_t* m12_pt, int32_t* m12_ls, uint8_t* inlier_pt, uint8_t* inlier_ls);
void plstvo_batch_free(PlContext* ctx, PlDeviceBatch* db);
int  plstvo_synchronize(PlContext* ctx);

/* pinned host memory for callers that want zero-staging H2D (e2e mode) */
void* plstvo_host_alloc(size_t bytes);
void  plstvo_host_free(void* p);

/* ---- instrumentation -------------------------------------------------------------------------- */
/* kernels launched by this library since the context was created (bench.py's gpu_launches) */
int64_t plstvo_launch_count(const PlContext* ctx);
/* device time of the two kernels of one pass over the resident batch, each launched alone `iters` times
 * on the context's stream and bracketed by CUDA events on that stream: *ms_match / *ms_solve = average
 * duration of one K1 (distance + top-2 and resolve kernels over the whole batch) / one K2 (track_solve, one CTA per
 * pair) launch.  n_tiles (optional) = matching problems the matcher works on (feature type enabled, both sides
 * non-empty); n_pairs (optional) = pairs. */
int     plstvo_batch_kernel_times(PlContext* ctx, PlDeviceBatch* db, int iters, double* ms_match,
                                  double* ms_solve, int32_t* n_tiles, int32_t* n_pairs);
/* The same per stage: ms[0] = the interval before the matcher (operands are expanded inside it: about 0), ms[1] = operand
 * expansion + distance + top-2 kernel, ms[2] = index resolution, ms[3] = building matched_pt / matched_ls when that is a
 * kernel of its own (the streamed solver; 0 when K2 does it internally), ms[4] = optimizePose (K2, or the streamed solver's
 * GN-loop / outlier / finalize kernels + K2 for the problems it hands back); of ms[4], streamed solver only (0 for K2):
 * ms[5] = the GN loop launch of stage 1, ms[6] = the gate + removeOutliers launch, ms[7] = the GN loop launch of stage 2.
 * counts (optional) = {bit 0: tensor-core matcher (always set), bit 1: streamed solver, bits 8..: problems the streamed solver handed to
 * the fp64 kernel in the last pass; work items of the distance kernel; matching problems; pairs}. */
int     plstvo_batch_stage_times(PlContext* ctx, PlDeviceBatch* db, int iters, double ms[8], int32_t counts[4]);
/* One solve pass over the resident batch (the matcher's output of the last pass is reused) with the solver kernels' cycle
 * counters switched on; it computes what the plain pass computes.  out: [B][PLSTVO_PHASE_SLOTS] clock64 sums per pair.
 * Slots [0, 8) are the fused kernel's phases (match-finalize, gather, GN eval, GN serial, gates/eigen, outliers, final,
 * sort+MAD), zero for pairs it did not solve.  Slots [8 + 11 s, 19 + 11 s) are the streamed solver's GN loop of stage s
 * (0 or 1), summed over the iterations of the pair's call: first-call record wait, evaluation, fold + store, barrier,
 * warp-0 sum and stop tests, close-call fp64 errors, 6x6 solve, increment + pose publish, trailing barriers, end-of-call
 * covariance, and then the iteration count; all zero where the stage did not run for the pair. */
#define PLSTVO_PHASE_SLOTS 32
int     plstvo_batch_phase_cycles(PlContext* ctx, PlDeviceBatch* db, int64_t* out);
/* GN evaluation (optimizeFunctions, src/stereoFrameHandler.cpp:549-694) of the resident matched
 * lists at given poses, streamed from HBM: the roofline kernel of config C5.
 * DT: [B][16]; H: [B][36]; g: [B][6]; e: [B]. */
int  plstvo_gn_eval_stream(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                           const PlMatchedBatch* matched, const double* DT, int iters,
                           double* H, double* g, double* e, float* ms_total);
/* test hook: the block-wide radix selection of the streamed solver's outlier pass (solve.cu: block_select_wide) on n_lists
 * caller-supplied lists (values[off[p] .. off[p+1])): out[p] = the k[p]-th smallest value (mode 0), or the k[p]-th smallest of
 * |x - pivot[p]| rounded to float (mode 1: the MAD form of src/auxiliar.cpp:399-402). */
int  plstvo_debug_select(PlContext* ctx, int n_lists, const int32_t* off, const double* values, const int32_t* k,
                         const double* pivot, int mode, double* out);
/* test hook: the intermediate words of the tensor-core matcher for the problems of a plstvo_match_batch call (same B, d1 /
 * off1, d2 / off2, nnr), after the same distance + top-2 and resolve kernels.  Per problem p, in problem order:
 *   rowp   [sum_p ceil(n2_p / 256) * n1_p]: the distance kernel's row words, [256-train block][n1] per problem: best distance
 *          over the block | second distance << 9 (511 = none) | candidate tag << 18 (parity | chunk group << 1 | lane << 4);
 *   colp   [sum_p n2_p]: column words, best | second << 9 | tag << 18 (the consumer warp, = (row % 128) / 16, of the best);
 *   rowkey [sum_p n1_p][2], colkey [sum_p n2_p][2]: the resolved keys (dist << 16 | index, dist2 << 16 | 0xFFFE), or
 *          0xFFFFFFFF as the second key when the other side has fewer than 2 rows.
 * A problem with an empty side has no words; its slots are left unchanged. */
int  plstvo_debug_tc_partials(PlContext* ctx, int B, const uint8_t* d1, const int32_t* off1, const uint8_t* d2,
                              const int32_t* off2, float nnr, uint32_t* rowp, uint32_t* colp, uint32_t* rowkey,
                              uint32_t* colkey);
/* test hook: both grey planes of the colour preparation a colour FLD session runs (the upload, then the remap and the
 * conversions of the same launch), on B pairs of host images img_l, img_r [B][height][width][channels] of a colour rectifier
 * rect.  rects (NULL, or [B] as plstvo_stereo_session_create_cams takes them, one per pair): pair b is prepared by rects[b]
 * instead of rect, a NULL entry or one without maps converting only.  Out, host, left images then right:
 *   grey [2][B][height][width]: cvtColor(remap(img), COLOR_BGR2GRAY), what ORB and LSD read (plstvo_rectify_batch's output);
 *   rgb  [2][B][height][width]: cvtColor(remap(img), COLOR_RGB2GRAY), what LBD reads on the FLD branch.
 * Without maps the remap is left out.  PLSTVO_E_INVALID (plstvo_last_error says which): a null pointer, B < 1, a rectifier
 * of another context, a grey rectifier, a table entry of another size or channel count than rect.  The call also updates
 * what plstvo_rectify_kernel_times reports. */
int  plstvo_debug_color_planes(PlContext* ctx, const PlRectifier* rect, const PlRectifier* const* rects, int B,
                               const uint8_t* img_l, const uint8_t* img_r, uint8_t* grey, uint8_t* rgb);
/* test hook for the on-chip 6x6 routines of the solver (ColPivHouseholderQR solve + log|det|, inverse, symmetric
 * eigenvalues) on n caller-supplied matrices: H [n][36] row-major, g [n][6] -> x [n][6], lad [n], inv [n][36], eig [n][6] */
int  plstvo_debug_algebra(PlContext* ctx, int n, const double* H, const double* g, double* x, double* lad,
                          double* inv, double* eig);
/* test hook for the device helpers both pose solvers use to decide and finish a problem, one warp per case, each run on
 * the same inputs:
 *   in  [n][PLSTVO_PH_IN]:  H[36] and g[6] (row-major; a solve), cov[36] (row-major; only its lower triangle is read),
 *                           DT[16], err, Tfw_prev[16], Tfw_cov_prev[36] (isGoodSolution and the pose finalisation),
 *                           xi[6] = [t; w] (expmap_se3), T[16] (inverse_se3, logmap_se3);
 *   out [n][PLSTVO_PH_OUT]: the Cholesky fast path with log|det| (x, lad, ok) and without it (x, ok), its all-register
 *                           copy on H's upper triangle (x, ok), the column-pivoted QR with log|det| (x, lad), the
 *                           isGoodSolution shortcut's verdict, isGoodSolution without and with the eigenvalues (verdict,
 *                           ascending eigenvalues), inverse_se3(T), logmap_se3(T), expmap_se3(xi), and the pose
 *                           finalisation on (DT, cov, err, Tfw_prev, Tfw_cov_prev): good, err_norm, DT, Tfw, Tfw_cov,
 *                           DT_cov_eig.  Flags are 0.0 / 1.0. */
#define PLSTVO_PH_IN_H 0
#define PLSTVO_PH_IN_G 36
#define PLSTVO_PH_IN_COV 42
#define PLSTVO_PH_IN_DT 78
#define PLSTVO_PH_IN_ERR 94
#define PLSTVO_PH_IN_TFW_PREV 95
#define PLSTVO_PH_IN_TFW_COV_PREV 111
#define PLSTVO_PH_IN_XI 147
#define PLSTVO_PH_IN_T 153
#define PLSTVO_PH_IN 169
#define PLSTVO_PH_CHOL_X 0
#define PLSTVO_PH_CHOL_LAD 6
#define PLSTVO_PH_CHOL_OK 7
#define PLSTVO_PH_CHOL0_X 8
#define PLSTVO_PH_CHOL0_OK 14
#define PLSTVO_PH_REGS_X 15
#define PLSTVO_PH_REGS_OK 21
#define PLSTVO_PH_QR_X 22
#define PLSTVO_PH_QR_LAD 28
#define PLSTVO_PH_SURELY 29
#define PLSTVO_PH_GOOD_FAST 30
#define PLSTVO_PH_GOOD_FULL 31
#define PLSTVO_PH_EIG 32
#define PLSTVO_PH_INV 38
#define PLSTVO_PH_LOG 54
#define PLSTVO_PH_EXP 60
#define PLSTVO_PH_FIN_GOOD 76
#define PLSTVO_PH_FIN_ERR 77
#define PLSTVO_PH_FIN_DT 78
#define PLSTVO_PH_FIN_TFW 94
#define PLSTVO_PH_FIN_TFW_COV 110
#define PLSTVO_PH_FIN_EIG 146
#define PLSTVO_PH_OUT 152
int  plstvo_debug_pose_helpers(PlContext* ctx, int n, const double* in, double* out);
/* test hook: one launch of the key-frame test a session run with the test runs after each step (needNewKF, then
 * currFrameIsKF where it fires), on n caller-placed streams.  Of results [n] only Tfw, DT and DT_cov are read; state [n] is
 * read and written back (the next call continues from it); out [n] receives each stream's PlKeyframeResult; priors [n]
 * (NULL: none read or returned) is read and written back, and a stream that fires has its Tfw and Tfw_cov set to I there.
 * k is not checked (NaN thresholds included), so that a test may place any value. */
int  plstvo_debug_keyframe(PlContext* ctx, const PlKeyframeConfig* k, int n, const PlPoseResult* results,
                           PlKeyframeState* state, PlKeyframeResult* out, PlPrior* priors);
/* POPC issue-rate micro-benchmark: returns 32-bit popcounts per second on this device */
int  plstvo_popc_rate(PlContext* ctx, double* popc_per_s);

#ifdef __cplusplus
}
#endif
#endif /* PLSTVO_H_ */
