// common.cuh — internal declarations shared by the sm_90a kernels and the C-ABI host code.
// Nothing here is part of the public boundary (include/plstvo.h is).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>

#include "../../include/plstvo.h"
#include "records.h"

namespace plstvo {

constexpr uint32_t KEY_NONE = 0xFFFFFFFFu;  // "no neighbour": larger than any (dist << 16 | idx) key

// ---- K1 work description --------------------------------------------------------------------------
// One matching problem = StVO::match(desc1, desc2) for one feature type of one frame pair
// (src/matching.cpp:63-91).  The matcher (match_tc.cu) leaves one resolved key pair per row (top-2 over all trains of
// each query) and one per column (top-2 over all queries of each train): both directions of the mutual check from ONE
// pass over the distances.
struct MatchProblem {
    const uint8_t* d1;     // [n1][32]
    const uint8_t* d2;     // [n2][32]
    int32_t n1, n2;
    int32_t enabled;       // 0: Config::hasPoints()/hasLines() false or an empty side -> all -1, no matcher work
    uint2*  rowpart;       // [n1]  (k1,k2) packed keys (dist << 16 | train index)
    uint2*  colpart;       // [n2]  (k1,k2) packed keys (dist << 16 | query index)
    int32_t* m12;          // [n1] result (problem-local train index or -1)
    float   nnr;
    int32_t best_lr;
};

// ---- K2 (track_solve) ------------------------------------------------------------------------------
constexpr int K2_THREADS = 512;   // one pair per SM at a time: at a few pairs per SM the per-pair latency is what counts
                                  // (128-thread CTAs x 4 per SM were measured: 3x the latency, same throughput at B = 512)
constexpr int K2_WARPS   = K2_THREADS / 32;
constexpr int ACC_N      = 28;    // 21 (upper triangle of J J^T w) + 6 (J r w) + 1 (r^2 w)

// The rows the solver reads (device copies, all frames or lists of a batch concatenated): a frame's records.h arrays
// (PlFrameBatch), or explicit matched lists (PlMatchedBatch: pt_pl and ls_le are the observations pl_obs and le_obs).  A
// null array is one not supplied (ls_level: level 0 everywhere; the inlier flags: all true).  Built by rows_dev (host.cuh).
struct RowsDev {
    const int32_t* pt_off;
    const int32_t* ls_off;
    const double*  pt_P;
    const double*  pt_pl;
    const double*  pt_sigma2;
    const uint8_t* pt_inlier;
    const double*  ls_sP;
    const double*  ls_eP;
    const double*  ls_le;
    const double*  ls_spl;
    const double*  ls_epl;
    const double*  ls_sigma2;
    const int32_t* ls_level;
    const uint8_t* ls_inlier;
};

struct SolveParams {
    PlCamera cam;
    PlConfig cfg;
    int32_t  mode;            // 0: track (match partials -> mutual -> gather -> optimizePose); 1: explicit lists
    int32_t  first_pair;      // pair index of blockIdx.x == 0
    RowsDev  prev, curr;      // mode 1: both the explicit lists (entry i's observation is current row i)
    const MatchProblem* problems;   // mode 0: [2 * pair + {0: points, 1: lines}]
    const PlPrior* priors;    // may be null
    PlPoseResult*  results;
    uint8_t* inlier_pt;       // mode 0: per prev feature; mode 1: per list entry
    uint8_t* inlier_ls;
    // feature storage: shared memory when it fits, else this global scratch (per CTA slice)
    double*  feat_scratch;
    size_t   feat_scratch_stride;  // doubles per CTA
    int32_t  cap_pt, cap_ls;  // capacity of the SoA arrays (max matched features per pair in this launch)
    int32_t  sort_cap;        // power of two >= max(cap_pt, cap_ls)
    int32_t  feat_in_smem;
    long long* phase_cycles;  // optional [pairs][PLSTVO_PHASE_SLOTS] cycle counters (plstvo_batch_phase_cycles), else null
    const int32_t* only_if;   // optional [pairs]: the CTA of pair p returns at once unless only_if[p] != 0
};

// ---- streamed optimizePose (solve.cu + gn_stream.cu): frames whose matched lists do not fit K2's shared memory ------------
// GN evaluations run as sweeps of gn_eval_stream_kernel over the fp32-packed records of ALL problems of the launch (HBM-bound),
// a one-warp-per-problem step kernel does the 6x6 solve / pose update / stop tests between sweeps, removeOutliers and the
// finalisation stay double precision on the fp64 lists.  Problems that leave the common path (robust fallback, solver_mode 1)
// are handed to K2 (global-scratch form) through SolveParams::only_if.
struct StreamCtl {            // per problem
    double DT0[16];           // initial pose of optimizePose
    double cov[36];
    double err, err_prev;
    int32_t iters, phase, fail_first, delegate, done, status, iters1, iters2, n_inl_p, n_inl_l, np, nl;
};
struct StreamBufs {
    float4*  rec_pt;          // 2 float4 per point slot, tile-planar (gn_stream.cu)
    float4*  rec_ls;          // 4 float4 per line slot
    int32_t* cnt_pt;          // [B] live records per problem
    int32_t* cnt_ls;
    double*  DT;              // [B][16] pose being optimised: read and updated by the GN loop kernel
    int32_t* active;          // [B]
    StreamCtl* ctl;           // [B]
    uint8_t* flag_pt;         // inlier flags per list entry (slots of the prev frame / of the explicit list)
    uint8_t* flag_ls;
    uint16_t* midx_pt;        // prev index of list entry k (track mode)
    uint16_t* midx_ls;
    int32_t* queue;           // problem queues of the persistent GN kernel (one int per launch of a solve: [2] per chunk)
    int32_t  sm_count;
};
// prm.feat_scratch must hold k2_feat_stride() doubles per pair; prm.feat_in_smem must be 0.  cams (optional, device): the
// camera of each pair, indexed by pair (prm.first_pair + p for the launch's pair p), instead of prm.cam; it selects the
// kernels' instantiations that read it (a separate kernel parameter, after the existing ones).
cudaError_t launch_stream_solve(const SolveParams& prm, int n_pairs, const StreamBufs& sb, cudaStream_t stream, int* launches,
                                cudaEvent_t* marks = nullptr,    // marks: 4 events (see solve.cu), instrumentation only
                                const PlCamera* cams = nullptr);

size_t k2_smem_bytes(int cap_pt, int cap_ls, int sort_cap, bool feat_in_smem);
size_t k2_feat_stride(int cap_pt, int cap_ls);   // doubles of global feature scratch per pair

// kernel launchers (defined in match.cu / solve.cu)
cudaError_t launch_match_finalize(const MatchProblem* problems, int n_problems, int max_n2, int32_t* counts,
                                  cudaStream_t stream);
cudaError_t launch_track_solve(const SolveParams& prm, int n_pairs, cudaStream_t stream, const PlCamera* cams = nullptr);
cudaError_t launch_select_selftest(const double* v, const int32_t* off, const int32_t* ks, const double* pivot, int mode, int n_lists,
                                   double* out, cudaStream_t stream);
cudaError_t launch_algebra_selftest(const double* H, const double* g, int n, double* x, double* lad, double* inv,
                                    double* eig, cudaStream_t stream);
cudaError_t launch_pose_helpers_selftest(const double* in, int n, double* out, cudaStream_t stream);
cudaError_t launch_popc_bench(uint32_t* out, int iters, int blocks, cudaStream_t stream);

// ---- StVO::matchGrid (match_grid.cu) ---------------------------------------------------------------------------
struct GridProblem {          // one frame: queries = left image, trains = right image
    int32_t n1, n2;
    const int32_t* q_cell;    // points: [n1][2]; lines: [n1][4] (sp.x, sp.y, ep.x, ep.y)
    const uint8_t* d1;
    const int32_t* t_cell;    // points: [n2][2]
    const double*  t_line;    // lines: [n2][4] in grid units
    const double*  t_dir;     // lines: [n2][2]
    const uint8_t* d2;
    int32_t* m12;             // [n1]
    int32_t* count;           // matches (or a negative error code)
    // scratch
    int32_t* grid_items;
    int2*    q_pairs;         // [n1][cap] (i2, d)
    int32_t* q_count;         // [n1]
    int32_t* t_count;         // [n2]
    int32_t* t_start;         // [n2 + 1]
    int32_t* t_slots;         // [n1 * cap]
    uint8_t* seen;            // [n1 * cap]
    int32_t* m21;             // [n2]
};
struct GridParams {
    int32_t rows, cols, cap, best_lr;
    PlGridWindow w;
    double ratio, line_sim_th;
};
size_t match_grid_smem_bytes(int rows, int cols);
cudaError_t launch_match_grid(const GridProblem* problems, int B, const GridParams& prm, bool lines, cudaStream_t stream);
// lift.cu: grid coordinates of raw key points / key lines (the loops in front of matchGrid, src/stereoFrame.cpp:129-139, :318-337)
cudaError_t launch_stereo_cells_points(int n_l, int n_r, double inv_w, double inv_h, const float* kp_l, const float* kp_r,
                                       int32_t* q_cell, int32_t* t_cell, cudaStream_t s);
cudaError_t launch_stereo_cells_lines(int n_l, int n_r, double inv_w, double inv_h, const float* seg_l, const float* seg_r,
                                      int32_t* q_line, double* t_line, double* t_dir, cudaStream_t s);
// lift.cu: stereo matches -> PointFeature / LineFeature records (src/stereoFrame.cpp:149-172, :348-397).  out: the device
// arrays PT_PL .. PT_SRC (points) or LS_SPL .. LS_SRC (lines), null entries skipped (all null: count only).
cudaError_t launch_lift_points(const PlCamera& cam, const PlStereoConfig& sc, int B, const int32_t* l_off, const float* kp_l,
                               const int32_t* oct_l, const uint8_t* desc_l, const int32_t* r_off, const float* kp_r,
                               const int32_t* m12, const RecPtrs& out, int32_t* counts, cudaStream_t s,
                               const int32_t* out_off = nullptr,    // out_off: compact output offsets per frame (else l_off)
                               const PlCamera* cams = nullptr);     // cams: device camera of each frame (else cam)
cudaError_t launch_lift_lines(const PlCamera& cam, const PlStereoConfig& sc, int B, const int32_t* l_off, const float* seg_l,
                              const float* ang_l, const int32_t* oct_l, const uint8_t* desc_l, const int32_t* r_off,
                              const float* seg_r, const int32_t* m12, const RecPtrs& out, int32_t* counts, cudaStream_t s,
                              const int32_t* out_off = nullptr, const PlCamera* cams = nullptr);

// orb.cu: ORB description (pyramid, blur, border filter, angle, rBRIEF) of a batch of images of one size
constexpr int ORB_MAX_LEVELS = 32;
struct OrbDevLevels {
    int n;                                   // levels
    int w[ORB_MAX_LEVELS], h[ORB_MAX_LEVELS];
    size_t raw_off[ORB_MAX_LEVELS];          // levels >= 1 in the resized-level buffer (level 0 is the input image)
    size_t blur_off[ORB_MAX_LEVELS];         // every level in the blurred-level buffer
    size_t raw_stride, blur_stride;          // bytes per image in either buffer
    float inv[ORB_MAX_LEVELS];               // 1.f / (float)pow(scale, l)
    float taps[7];                           // getGaussianKernel(7, 2, CV_32F)
};
cudaError_t orb_upload_tables();             // pattern and disc tables into the current device's constant memory
cudaError_t launch_orb(const OrbDevLevels& L, int n_img, int W, int H, int edge, const uint8_t* images, uint8_t* raw_pyr,
                       uint8_t* blur_pyr, const int32_t* const* rs_tab, const int32_t* kp_off, int n_rows, const float* kp_xy,
                       const int32_t* kp_oct, const float* kp_angle, int32_t* src_idx, int32_t* counts, float* out_angle,
                       uint8_t* out_desc, cudaStream_t s, cudaEvent_t* ev, int* launches);
// the two halves of launch_orb that key-point selection sits between
void launch_orb_pyramid(const OrbDevLevels& L, int n_img, const uint8_t* images, uint8_t* raw_pyr, uint8_t* blur_pyr,
                        const int32_t* const* rs_tab, cudaStream_t s, int* launches);
void launch_orb_describe(const OrbDevLevels& L, int n_img, const uint8_t* images, const uint8_t* raw_pyr,
                         const uint8_t* blur_pyr, const int32_t* kp_off, int n_rows, const float* kp_xy, const int32_t* kp_oct,
                         const float* kp_angle, const int32_t* src_idx, const int32_t* counts, float* out_angle,
                         uint8_t* out_desc, cudaStream_t s, int* launches);

// ORB key-point selection (cv::ORB's computeKeyPoints with an empty mask).  Rows: the levels of one image stacked, level l's
// row y is row row0[l] + y; key points come out per image in (level, y, x) order.
struct OrbDetectLevels {
    int keep1[ORB_MAX_LEVELS];        // retainBest count on the FAST score: n_l (FAST_SCORE) or 2 n_l (HARRIS_SCORE)
    int keep2[ORB_MAX_LEVELS];        // retainBest count on the Harris response: n_l
    int row0[ORB_MAX_LEVELS + 1];     // prefix of the level heights; row0[n] = rows per image
    float layer_scale[ORB_MAX_LEVELS];// (float)pow(scale, l): pt = level coordinate * layer_scale
    int edge;                         // runByImageBorder on the level
    float harris_scale4;              // (1 / (4 * 7 * 255))^4, multiplied in float as OpenCV does
};
// FAST + NMS + border filter into the score maps (blur_pyr's geometry) with a 256-bin histogram per (image, level), the
// per-(image, level) FAST cut, row counts, per-image row scan and image offsets (sel_off [n_img + 1], sel_cnt [n_img]).
void launch_orb_fast_select(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, const uint8_t* images,
                            const uint8_t* raw_pyr, const int32_t* fast_th, uint8_t* score, uint32_t* hist, int32_t* cut,
                            int32_t* row_cnt, int32_t* row_base, int32_t* img_cnt, int32_t* sel_off, cudaStream_t s,
                            cudaEvent_t ev_fast_done, int* launches);
// writes the FAST-selected key points densely at sel_off[img] + rank: level coordinates, pt, octave, FAST response, rank
void launch_orb_fast_write(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, const uint8_t* score, const int32_t* cut,
                           const int32_t* row_base, const int32_t* sel_off, int2* lxy, float* xy, int32_t* oct, float* resp,
                           int32_t* rank, cudaStream_t s, int* launches);
// HARRIS_SCORE: responses of the FAST-selected candidates, the n_l-th largest per (image, level), and the survivors densely
// at out_off[img] + rank (out_off [n_img + 1], out_cnt [n_img])
void launch_orb_harris_select(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, int n_cand, const uint8_t* images,
                              const uint8_t* raw_pyr, const int32_t* row_base, const int32_t* sel_off, const int2* lxy,
                              const int32_t* oct, float* hresp, uint32_t* cut_key, int32_t* lvl_keep, int32_t* out_off,
                              int32_t* out_cnt, cudaStream_t s, int* launches);
void launch_orb_harris_write(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, const int32_t* sel_off,
                             const float* xy, const int32_t* oct, const float* hresp, const uint32_t* cut_key,
                             const int32_t* out_off, float* out_xy, int32_t* out_oct, float* out_resp, int32_t* out_rank,
                             cudaStream_t s, int* launches);

__device__ __forceinline__ float fast_atan2(float y, float x) {   // cv::fastAtan2, unfused like OpenCV's build
    constexpr float deg = (float)(180 / 3.14159265358979323846);
    constexpr float p1 = 0.9997878412794807f * deg, p3 = -0.3258083974640975f * deg, p5 = 0.1555786518463281f * deg,
                    p7 = -0.04432655554792128f * deg;
    const float ax = fabsf(x), ay = fabsf(y), eps = (float)2.2204460492503131e-16;
    float a, c, c2;
    const bool wide = ax >= ay;
    c = wide ? __fdiv_rn(ay, __fadd_rn(ax, eps)) : __fdiv_rn(ax, __fadd_rn(ay, eps));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    if (!wide) a = __fsub_rn(90.f, a);
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

// lsd.cu: LSD line segments (cv::LineSegmentDetector, LSD_REFINE_NONE) on a batch of grey images of one size
constexpr int LSD_GRAD_MAX = 510;                      // |gx|, |gy| of the 2x2 gradient
constexpr int LSD_TRIG_SIDE = 2 * LSD_GRAD_MAX + 1;    // trig table: code = (gx + 510) * 1021 + (gy + 510)
constexpr int LSD_MAX_KH = 15;                         // blur half-width
struct LsdTaps { int kh; int t[2 * LSD_MAX_KH + 1]; };   // GaussianBlur's fixed-point taps (8 fractional bits)
struct LsdRegion { double cx, cy, theta; int32_t start, count; };   // a kept region: centroid, angle, its pixels in rpix
struct LsdLaunch {
    int n_img, W, H, w, h;         // input size, scaled size
    double scale, rho, prec;       // scale, gradient threshold quant / sin(prec), angle tolerance (radians)
    int min_reg, reg_cap, n_bins;  // smallest kept region, region records per image, bins
    LsdTaps taps;
    const uint8_t* images;         // [n_img][H][W]
    uint8_t *blurred, *scaled;     // [n_img][H][W], [n_img][h][w] (unused where scale == 1; scaled unused where w, h == W, H)
    uint8_t* scratch;              // lsd_scratch_bytes(n_img, w, h)
    unsigned long long* max_bits;  // [n_img]
    int32_t *hist, *n_seeds;       // [n_img][n_bins], [n_img]
    const float4* trig;            // [LSD_TRIG_SIDE^2]: (float)cos, (float)sin of the angle; cosf, sinf of (float)angle
    LsdRegion* regions;            // [n_img][reg_cap]
    int32_t* n_regions;            // [n_img]
};
size_t lsd_scratch_bytes(int n_img, int w, int h);
// ev[0..3]: start, blur + resize, gradient + seed order, region growing
cudaError_t launch_lsd_grow(const LsdLaunch& L, cudaStream_t s, cudaEvent_t* ev, int* launches);
// regions r_off[i] .. r_off[i + 1] of image i (n_reg in all), dir [n_reg] (cos, sin) of their angles -> seg [n_reg]
cudaError_t launch_lsd_extent(const LsdLaunch& L, int n_reg, const int32_t* r_off, const double2* dir, float4* seg,
                              cudaStream_t s, int* launches);

// lbd.cu: LBD descriptors of given octave-0 key lines (BinaryDescriptor::compute, default Params) on a batch of images
cudaError_t lbd_upload_tables(const float* coef_g, const float* coef_l);   // (float)gaussCoefG_ [63], (float)gaussCoefL_ [21]
cudaError_t launch_lbd(int n_img, int W, int H, const uint8_t* images, const int32_t* kl_off, int n_lines, const float* seg,
                       const float2* dir, const int32_t* npix, short2* grad, uint8_t* out_desc, cudaStream_t s,
                       cudaEvent_t* ev, int* launches);   // dir: (cosf, sinf) of each angle; ev[0..2]: start, gradients, descriptors

// rectify.cu: cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of n_img grey W x H images on CV_16SC2 + CV_16UC1 maps; image z takes
// the right maps (m1[1], m2[1]) where (z / per_block) is odd, the left ones otherwise.  With a map table (device, [per_block][2])
// image z takes maps[2 (z % per_block) + side] instead, and an entry with null maps is copied.
struct RemapMaps {
    const short2* m1;
    const uint16_t* m2;
};
cudaError_t launch_rectify_remap(int n_img, int per_block, int W, int H, const uint8_t* src, uint8_t* dst,
                                 const short2* const m1[2], const uint16_t* const m2[2], cudaStream_t s, int* launches,
                                 const RemapMaps* maps = nullptr);

// GN evaluation streamed from HBM (roofline kernel of config C5): fp32-packed records, TMA-staged tiles
int gn_stream_tiles(int n_pt, int n_ls);
int gn_stream_partials_per_slice();   // fp64 partial records one slice writes (one per consumer warp)   // 16 KB tiles of one problem (512 points or 256 lines each)
cudaError_t launch_pack_records(const RowsDev& m, const PlCamera& cam, int B, int n_pt, int n_ls, float4* pt, float4* ls,
                                cudaStream_t stream);
cudaError_t launch_gn_eval_stream(const PlCamera& cam, const PlConfig& cfg, const int32_t* pt_off, const int32_t* ls_off,
                                  const float4* pt, const float4* ls, int B, const double* DT, double* partial,
                                  int slices_per_problem, int sm_count, double* H, double* g, double* e, cudaStream_t stream);

// cudaFuncSetAttribute is per device: a process may drive several GPUs (one context each), so the opted-in dynamic
// shared-memory size is remembered per device (`done`: one slot per device ordinal, zero-initialised by the caller).
inline cudaError_t ensure_dynamic_smem(const void* fn, size_t bytes, size_t* done /* [64] */) {
    static std::mutex mu;   // the caches are per function, contexts (and their locks) are per device: two contexts on one
    std::lock_guard<std::mutex> lock(mu);   // device may launch the same kernel concurrently
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    size_t& have = done[dev & 63];
    if (bytes <= have) return cudaSuccess;
    e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) have = bytes;
    return e;
}

// ---- PTX helpers: mbarrier + 1-D bulk async copy (TMA engine, UBLKCP in SASS) ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar /* shared address */, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait(smem_u32(bar), parity); }
// global -> shared bulk copy completing on an mbarrier; addresses and size must be multiples of 16 B
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

}  // namespace plstvo
