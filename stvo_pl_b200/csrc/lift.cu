// lift.cu — 3-D lifting of the stereo matches (SURVEY 8(f)-2): src/stereoFrame.cpp:149-172 (points), :348-397 (lines),
// filterLineSegmentDisparity :405-415, lineSegmentOverlapStereo :473-508, backProjection
// src/pinholeStereoCamera.cpp:221-229, sigma2 from the pyramid level src/stereoFeatures.cpp:41-47, :107-115.
// One CTA per frame: every thread evaluates the filters of its matches, an ordered block scan compacts the survivors
// (ascending left index, like the reference's push_back loop), then the records and the surviving descriptor rows are
// written densely.  Multiplications and additions that the compiler could contract into FMAs are spelled with the
// round-to-nearest intrinsics, so the records are bit-identical to the reference's SSE2 arithmetic.
#include "common.cuh"

namespace plstvo {

namespace {

constexpr int LF_THREADS = 256;

__device__ __forceinline__ double sigma2_of_level(int level, double scale) {
    double s = 1.0;
    for (int i = 0; i < level; i++) s = __dmul_rn(s, scale);
    return 1.0 / __dmul_rn(s, s);
}

__device__ __forceinline__ void back_projection(const PlCamera& c, double u, double v, double disp, double* P) {
    const double bd = c.b / disp;
    P[0] = __dmul_rn(bd, u - c.cx);
    P[1] = __dmul_rn(bd, v - c.cy);
    P[2] = __dmul_rn(bd, c.fx);
}

__device__ __forceinline__ double overlap_stereo(const PlStereoConfig& sc, double spl_obs, double epl_obs, double spl_proj,
                                                 double epl_proj) {   // :473-508
    double overlap = 1.0;
    if (fabs(epl_obs - spl_obs) > sc.line_horiz_th) {
        const double sln = (epl_obs < spl_obs) ? epl_obs : spl_obs, eln = (spl_obs < epl_obs) ? epl_obs : spl_obs;
        const double spn = (epl_proj < spl_proj) ? epl_proj : spl_proj, epn = (spl_proj < epl_proj) ? epl_proj : spl_proj;
        const double length = eln - spn;
        if ((epn < sln) || (spn > eln)) overlap = 0.0;
        else if ((epn > eln) && (spn < sln)) overlap = eln - sln;
        else overlap = ((epn < eln) ? epn : eln) - ((sln < spn) ? spn : sln);
        if (length > (double)0.01f) overlap = overlap / length;
        else overlap = 0.0;
        if (overlap > 1.0) overlap = 1.0;
    }
    return overlap;
}

// ordered compaction helper: exclusive scan of one flag per thread over the block, running base across rounds
__device__ int block_scan_flag(int flag, int* s_warp, int* s_base, int* total_round) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, flag);
    const int within = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int before = 0, tot = 0;
    for (int w = 0; w < LF_THREADS / 32; w++) {
        if (w < warp) before += s_warp[w];
        tot += s_warp[w];
    }
    const int pos = *s_base + before + within;
    __syncthreads();
    if (tid == 0) *s_base += tot;
    *total_round = tot;
    __syncthreads();
    return pos;
}

// CAMS: frame f is back-projected under cams[f], else under cam.
template <bool CAMS>
__global__ void __launch_bounds__(LF_THREADS)
lift_points_kernel(PlCamera cam, PlStereoConfig sc, const int32_t* __restrict__ l_off, const float* __restrict__ kp_l,
                   const int32_t* __restrict__ oct_l, const uint8_t* __restrict__ desc_l, const int32_t* __restrict__ r_off,
                   const float* __restrict__ kp_r, const int32_t* __restrict__ m12, double* pt_pl, double* pt_disp,
                   double* pt_P, double* pt_sigma2, int32_t* pt_level, uint8_t* pdesc_out, int32_t* src_idx,
                   int32_t* counts, const int32_t* __restrict__ out_off, const PlCamera* __restrict__ cams) {
    // out_off == nullptr: frame f's records start at element l_off[f] of every output; else at out_off[f] (compact layout).
    // Output pointers may be null (not wanted); with all of them null the kernel only counts.
    __shared__ int s_warp[LF_THREADS / 32], s_base;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int a0 = l_off[f], n = l_off[f + 1] - a0, b0 = r_off[f];
    const size_t o0 = out_off ? (size_t)out_off[f] : (size_t)a0;
    if constexpr (CAMS) cam = cams[f];
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int base = 0; base < n; base += LF_THREADS) {
        const int i1 = base + tid;
        int keep = 0;
        double disp = 0.0;
        if (i1 < n) {
            const int i2 = m12[a0 + i1];
            if (i2 >= 0) {
                const float yl = kp_l[2 * (size_t)(a0 + i1) + 1], yr = kp_r[2 * (size_t)(b0 + i2) + 1];
                if ((double)fabsf(__fsub_rn(yl, yr)) <= sc.max_dist_epip) {                        // :156
                    disp = (double)__fsub_rn(kp_l[2 * (size_t)(a0 + i1)], kp_r[2 * (size_t)(b0 + i2)]);   // float - float
                    keep = (disp >= sc.min_disp) ? 1 : 0;                                           // :159
                }
            }
        }
        int tot;
        const int k = block_scan_flag(keep, s_warp, &s_base, &tot);
        if (keep) {
            const size_t o = o0 + k, src = (size_t)a0 + i1;
            const double u = (double)kp_l[2 * src], v = (double)kp_l[2 * src + 1];
            if (pt_pl) {
                pt_pl[2 * o] = u;
                pt_pl[2 * o + 1] = v;
            }
            if (pt_disp) pt_disp[o] = disp;
            if (pt_P) back_projection(cam, u, v, disp, pt_P + 3 * o);
            if (pt_level) pt_level[o] = oct_l[src];
            if (pt_sigma2) pt_sigma2[o] = sigma2_of_level(oct_l[src], sc.orb_scale_factor);
            if (src_idx) src_idx[o] = i1;
            if (pdesc_out) {
                const uint4* d = reinterpret_cast<const uint4*>(desc_l + src * 32);
                uint4* q = reinterpret_cast<uint4*>(pdesc_out + o * 32);
                q[0] = d[0];
                q[1] = d[1];
            }
        }
        __syncthreads();   // a later round may overwrite rows this round still reads (o <= src always, rounds ascend)
    }
    if (tid == 0) counts[f] = s_base;
}

template <bool CAMS>
__global__ void __launch_bounds__(LF_THREADS)
lift_lines_kernel(PlCamera cam, PlStereoConfig sc, const int32_t* __restrict__ l_off, const float* __restrict__ seg_l,
                  const float* __restrict__ ang_l, const int32_t* __restrict__ oct_l, const uint8_t* __restrict__ desc_l,
                  const int32_t* __restrict__ r_off, const float* __restrict__ seg_r, const int32_t* __restrict__ m12,
                  double* ls_spl, double* ls_epl, double* ls_sdisp, double* ls_edisp, double* ls_sP, double* ls_eP,
                  double* ls_le, double* ls_angle, double* ls_sigma2, int32_t* ls_level, uint8_t* ldesc_out,
                  int32_t* src_idx, int32_t* counts, const int32_t* __restrict__ out_off,
                  const PlCamera* __restrict__ cams) {
    __shared__ int s_warp[LF_THREADS / 32], s_base;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int a0 = l_off[f], n = l_off[f + 1] - a0, b0 = r_off[f];
    const size_t o0 = out_off ? (size_t)out_off[f] : (size_t)a0;
    if constexpr (CAMS) cam = cams[f];
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int base = 0; base < n; base += LF_THREADS) {
        const int i1 = base + tid;
        int keep = 0;
        double spl[2] = {0, 0}, epl[2] = {0, 0}, le[3] = {0, 0, 0}, disp_s = 0, disp_e = 0;
        if (i1 < n) {
            const int i2 = m12[a0 + i1];
            if (i2 >= 0) {
                const float* L = seg_l + 4 * (size_t)(a0 + i1);
                const float* R = seg_r + 4 * (size_t)(b0 + i2);
                spl[0] = L[0]; spl[1] = L[1]; epl[0] = L[2]; epl[1] = L[3];
                le[0] = spl[1] - epl[1];                                                   // sp_l x ep_l (:357)
                le[1] = epl[0] - spl[0];
                le[2] = __dsub_rn(__dmul_rn(spl[0], epl[1]), __dmul_rn(spl[1], epl[0]));
                const double nrm = sqrt(__dadd_rn(__dmul_rn(le[0], le[0]), __dmul_rn(le[1], le[1])));
                le[0] /= nrm; le[1] /= nrm; le[2] /= nrm;
                double spr[2] = {R[0], R[1]}, epr[2] = {R[2], R[3]};
                const double overlap = overlap_stereo(sc, spl[1], epl[1], spr[1], epr[1]);   // :362
                // :366-367: sp_r is overwritten coefficient by coefficient, ep_r is then computed from the UPDATED sp_r
                spr[0] = __dadd_rn(__dmul_rn(spr[0], spl[1] - epr[1]), __dmul_rn(epr[0], spr[1] - spl[1])) / (spr[1] - epr[1]);
                spr[1] = spl[1];
                epr[0] = __dadd_rn(__dmul_rn(spr[0], epl[1] - epr[1]), __dmul_rn(epr[0], spr[1] - epl[1])) / (spr[1] - epr[1]);
                epr[1] = epl[1];
                disp_s = spl[0] - spr[0];                                                   // :405-415
                disp_e = epl[0] - epr[0];
                const double mn = (disp_e < disp_s) ? disp_e : disp_s, mx = (disp_s < disp_e) ? disp_e : disp_s;
                if (mn / mx < sc.ls_min_disp_ratio) { disp_s = -1.0; disp_e = -1.0; }
                keep = (disp_s >= sc.min_disp && disp_e >= sc.min_disp && fabs(spl[1] - epl[1]) > sc.line_horiz_th &&
                        fabs(spr[1] - epr[1]) > sc.line_horiz_th && overlap > sc.stereo_overlap_th) ? 1 : 0;   // :371-374
            }
        }
        int tot;
        const int k = block_scan_flag(keep, s_warp, &s_base, &tot);
        if (keep) {
            const size_t o = o0 + k, src = (size_t)a0 + i1;
            if (ls_sP) back_projection(cam, spl[0], spl[1], disp_s, ls_sP + 3 * o);
            if (ls_eP) back_projection(cam, epl[0], epl[1], disp_e, ls_eP + 3 * o);
            if (ls_spl) { ls_spl[2 * o] = spl[0]; ls_spl[2 * o + 1] = spl[1]; }
            if (ls_epl) { ls_epl[2 * o] = epl[0]; ls_epl[2 * o + 1] = epl[1]; }
            if (ls_sdisp) ls_sdisp[o] = disp_s;
            if (ls_edisp) ls_edisp[o] = disp_e;
            if (ls_le) { ls_le[3 * o] = le[0]; ls_le[3 * o + 1] = le[1]; ls_le[3 * o + 2] = le[2]; }
            if (ls_angle) ls_angle[o] = (double)ang_l[src];
            if (ls_level) ls_level[o] = oct_l[src];
            if (ls_sigma2) ls_sigma2[o] = sigma2_of_level(oct_l[src], sc.lsd_scale);
            if (src_idx) src_idx[o] = i1;
            if (ldesc_out) {
                const uint4* d = reinterpret_cast<const uint4*>(desc_l + src * 32);
                uint4* q = reinterpret_cast<uint4*>(ldesc_out + o * 32);
                q[0] = d[0];
                q[1] = d[1];
            }
        }
        __syncthreads();
    }
    if (tid == 0) counts[f] = s_base;
}

// grid coordinates of the raw stereo features (src/stereoFrame.cpp:129-139 points; :318-337 lines): the caller-side loops
// that feed matchGrid.  float coordinate x double inverse cell size, truncated toward zero for the integer cells.
__global__ void stereo_cells_points_kernel(int n_l, int n_r, double inv_w, double inv_h, const float* __restrict__ kp_l,
                                           const float* __restrict__ kp_r, int32_t* __restrict__ q_cell,
                                           int32_t* __restrict__ t_cell) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_l) {
        q_cell[2 * i] = (int)((double)kp_l[2 * i] * inv_w);
        q_cell[2 * i + 1] = (int)((double)kp_l[2 * i + 1] * inv_h);
    }
    if (i < n_r) {
        t_cell[2 * i] = (int)((double)kp_r[2 * i] * inv_w);
        t_cell[2 * i + 1] = (int)((double)kp_r[2 * i + 1] * inv_h);
    }
}

__global__ void stereo_cells_lines_kernel(int n_l, int n_r, double inv_w, double inv_h, const float* __restrict__ seg_l,
                                          const float* __restrict__ seg_r, int32_t* __restrict__ q_line,
                                          double* __restrict__ t_line, double* __restrict__ t_dir) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_l) {
#pragma unroll
        for (int k = 0; k < 4; k++) q_line[4 * i + k] = (int)((double)seg_l[4 * i + k] * ((k & 1) ? inv_h : inv_w));
    }
    if (i < n_r) {
        const float sx = seg_r[4 * i], sy = seg_r[4 * i + 1], ex = seg_r[4 * i + 2], ey = seg_r[4 * i + 3];
        t_line[4 * i] = (double)sx * inv_w;
        t_line[4 * i + 1] = (double)sy * inv_h;
        t_line[4 * i + 2] = (double)ex * inv_w;
        t_line[4 * i + 3] = (double)ey * inv_h;
        const double vx = (double)__fsub_rn(ex, sx) * inv_w, vy = (double)__fsub_rn(ey, sy) * inv_h;   // float - float (:332)
        const double mag = sqrt(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));                     // include/matching.h:43-48
        t_dir[2 * i] = vx / mag;
        t_dir[2 * i + 1] = vy / mag;
    }
}

}  // namespace

cudaError_t launch_stereo_cells_points(int n_l, int n_r, double inv_w, double inv_h, const float* kp_l, const float* kp_r,
                                       int32_t* q_cell, int32_t* t_cell, cudaStream_t s) {
    const int n = n_l > n_r ? n_l : n_r;
    if (n <= 0) return cudaSuccess;
    stereo_cells_points_kernel<<<(n + 255) / 256, 256, 0, s>>>(n_l, n_r, inv_w, inv_h, kp_l, kp_r, q_cell, t_cell);
    return cudaGetLastError();
}

cudaError_t launch_stereo_cells_lines(int n_l, int n_r, double inv_w, double inv_h, const float* seg_l, const float* seg_r,
                                      int32_t* q_line, double* t_line, double* t_dir, cudaStream_t s) {
    const int n = n_l > n_r ? n_l : n_r;
    if (n <= 0) return cudaSuccess;
    stereo_cells_lines_kernel<<<(n + 255) / 256, 256, 0, s>>>(n_l, n_r, inv_w, inv_h, seg_l, seg_r, q_line, t_line, t_dir);
    return cudaGetLastError();
}

cudaError_t launch_lift_points(const PlCamera& cam, const PlStereoConfig& sc, int B, const int32_t* l_off, const float* kp_l,
                               const int32_t* oct_l, const uint8_t* desc_l, const int32_t* r_off, const float* kp_r,
                               const int32_t* m12, const RecPtrs& out, int32_t* counts, cudaStream_t s, const int32_t* out_off,
                               const PlCamera* cams) {
    if (B <= 0) return cudaSuccess;
    const auto kernel = cams ? lift_points_kernel<true> : lift_points_kernel<false>;
    kernel<<<B, LF_THREADS, 0, s>>>(cam, sc, l_off, kp_l, oct_l, desc_l, r_off, kp_r, m12, out.at<double>(PT_PL),
                                    out.at<double>(PT_DISP), out.at<double>(PT_P), out.at<double>(PT_S2),
                                    out.at<int32_t>(PT_LEVEL), out.at<uint8_t>(PT_DESC), out.at<int32_t>(PT_SRC), counts,
                                    out_off, cams);
    return cudaGetLastError();
}

cudaError_t launch_lift_lines(const PlCamera& cam, const PlStereoConfig& sc, int B, const int32_t* l_off, const float* seg_l,
                              const float* ang_l, const int32_t* oct_l, const uint8_t* desc_l, const int32_t* r_off,
                              const float* seg_r, const int32_t* m12, const RecPtrs& out, int32_t* counts, cudaStream_t s,
                              const int32_t* out_off, const PlCamera* cams) {
    if (B <= 0) return cudaSuccess;
    const auto kernel = cams ? lift_lines_kernel<true> : lift_lines_kernel<false>;
    kernel<<<B, LF_THREADS, 0, s>>>(cam, sc, l_off, seg_l, ang_l, oct_l, desc_l, r_off, seg_r, m12, out.at<double>(LS_SPL),
                                    out.at<double>(LS_EPL), out.at<double>(LS_SDISP), out.at<double>(LS_EDISP),
                                    out.at<double>(LS_SP), out.at<double>(LS_EP), out.at<double>(LS_LE),
                                    out.at<double>(LS_ANGLE), out.at<double>(LS_S2), out.at<int32_t>(LS_LEVEL),
                                    out.at<uint8_t>(LS_DESC), out.at<int32_t>(LS_SRC), counts, out_off, cams);
    return cudaGetLastError();
}

}  // namespace plstvo
