// orb.cu — ORB description on the GPU (SURVEY 8(f)-4, the half of cv::ORB that runs after key-point selection):
// image pyramid, border filter, intensity-centroid angle and rotated BRIEF, bit-identical to OpenCV 4.13's
// ORB::compute / ORB::detectAndCompute for the key points given.  Batched over n images of one size (the left and right
// images of B stereo frames).  How each stage rounds: level sizes cvRound(W * (1.f / (float)s^l)), INTER_LINEAR_EXACT from
// the level above; the border filter tests cvRound(pt); the blur is sepFilter2D's float path (ORB blurs a sub-matrix of its
// pyramid buffer); angles and rotated pattern points follow orb.cpp in float.  Float arithmetic is spelled with the _rn intrinsics; where OpenCV's own build fuses (the vector code of the
// blur, in its FMA dispatch) with __fmaf_rn.
//
// Kernels (one launch each per level where marked):
//   orb_resize_kernel    per level >= 1   INTER_LINEAR_EXACT from the level above, 64x16 output tile, source tile in smem
//   orb_blur_kernel      per level        GaussianBlur 7x7 sigma 2 (float path), 64x16 output tile + 3-pixel halo in smem
//   orb_filter_kernel    one CTA / image  border filter as an ordered compaction (survivors keep input order)
//   orb_describe_kernel  one warp / row   angle (if not given) by warp reduction of the moments, then 8 comparisons per
//                                         lane and one __ballot_sync per 32-bit descriptor word
// Key-point selection (plstvo_orb_detect_and_compute_batch), between the pyramid and the describe kernel:
//   orb_fast_kernel        per level      FAST-9/16 score, 3x3 NMS, level border filter: u8 score map + 256-bin histogram per
//                                         (image, level); 64x16 output tile + 4-pixel halo in smem
//   orb_fast_cut_kernel    one thread / (image, level)   retainBest on the FAST score as a cut on the histogram
//   orb_fast_rows_kernel   one warp / row of the stacked levels   count (then, after the scans, write) the kept points
//   orb_row_scan_kernel    one CTA / image   row offsets;  orb_offsets_kernel  one CTA   per-image offsets
//   orb_harris_kernel      one thread / candidate   HARRIS_SCORE: the response on the raw level
//   orb_harris_cut_kernel  one CTA / (image, level)   the n_l-th largest response by radix selection
//   orb_harris_write_kernel  one CTA / image   ordered compaction of the responses >= the cut
#include "common.cuh"
#include "orb_pattern.h"

namespace plstvo {

namespace orb {   // named (not anonymous): the kernels keep stable symbol names across builds

constexpr int TILE_W = 64, TILE_H = 16, THREADS = 256;
constexpr int RS_ROWS = 40, RS_COLS = 160;   // staged source tile of the resize (covers scale factors up to 2)

__constant__ signed char c_pattern[256][4];
__constant__ int c_umax[16];

__device__ __forceinline__ int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

__device__ __forceinline__ const uint8_t* raw_level(const OrbDevLevels& L, const uint8_t* images, const uint8_t* raw_pyr,
                                                    int img, int l) {
    return l == 0 ? images + (size_t)img * L.w[0] * L.h[0] : raw_pyr + (size_t)img * L.raw_stride + L.raw_off[l];
}

__global__ void __launch_bounds__(THREADS)
orb_resize_kernel(OrbDevLevels L, int l, const uint8_t* __restrict__ images, uint8_t* raw_pyr,
                  const int32_t* __restrict__ xtab, const int32_t* __restrict__ ytab) {
    // xtab / ytab: [2 * dw] / [2 * dh]: source offset, then the 8-bit weight of the second tap (0: the edge pixel alone)
    __shared__ uint8_t s_src[RS_ROWS][RS_COLS];
    const int img = blockIdx.z, sw = L.w[l - 1], sh = L.h[l - 1], dw = L.w[l], dh = L.h[l];
    const uint8_t* src = raw_level(L, images, raw_pyr, img, l - 1);
    uint8_t* dst = raw_pyr + (size_t)img * L.raw_stride + L.raw_off[l];
    const int x0 = blockIdx.x * TILE_W, y0 = blockIdx.y * TILE_H;
    const int x1 = min(x0 + TILE_W, dw) - 1, y1 = min(y0 + TILE_H, dh) - 1;
    const int c0 = xtab[x0], r0 = ytab[y0];
    const int c1 = min(xtab[x1] + 1, sw - 1), r1 = min(ytab[y1] + 1, sh - 1);
    const bool staged = (r1 - r0 + 1) <= RS_ROWS && (c1 - c0 + 1) <= RS_COLS;
    if (staged) {
        const int nc = c1 - c0 + 1, n = (r1 - r0 + 1) * nc;
        for (int i = threadIdx.x; i < n; i += THREADS) s_src[i / nc][i % nc] = src[(size_t)(r0 + i / nc) * sw + c0 + i % nc];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TILE_W * TILE_H; i += THREADS) {
        const int x = x0 + (i % TILE_W), y = y0 + (i / TILE_W);
        if (x >= dw || y >= dh) continue;
        const int xo = xtab[x], xc = xtab[dw + x], yo = ytab[y], yc = ytab[dh + y];
        const int xa = xo, xb = xo + (xc ? 1 : 0), ya = yo, yb = yo + (yc ? 1 : 0);
        uint32_t p00, p01, p10, p11;
        if (staged) {
            p00 = s_src[ya - r0][xa - c0]; p01 = s_src[ya - r0][xb - c0];
            p10 = s_src[yb - r0][xa - c0]; p11 = s_src[yb - r0][xb - c0];
        } else {
            p00 = src[(size_t)ya * sw + xa]; p01 = src[(size_t)ya * sw + xb];
            p10 = src[(size_t)yb * sw + xa]; p11 = src[(size_t)yb * sw + xb];
        }
        const uint32_t h0 = (256u - xc) * p00 + (uint32_t)xc * p01, h1 = (256u - xc) * p10 + (uint32_t)xc * p11;
        dst[(size_t)y * dw + x] = (uint8_t)((h0 * (256u - yc) + h1 * (uint32_t)yc + 0x8000u) >> 16);
    }
}

__global__ void __launch_bounds__(THREADS)
orb_blur_kernel(OrbDevLevels L, int l, const uint8_t* __restrict__ images, const uint8_t* __restrict__ raw_pyr,
                uint8_t* blur_pyr) {
    __shared__ uint8_t s_in[TILE_H + 6][TILE_W + 6];
    __shared__ float s_row[TILE_H + 6][TILE_W];
    const int img = blockIdx.z, w = L.w[l], h = L.h[l];
    const uint8_t* src = raw_level(L, images, raw_pyr, img, l);
    uint8_t* dst = blur_pyr + (size_t)img * L.blur_stride + L.blur_off[l];
    const int x0 = blockIdx.x * TILE_W, y0 = blockIdx.y * TILE_H;
    for (int i = threadIdx.x; i < (TILE_H + 6) * (TILE_W + 6); i += THREADS) {
        const int ty = i / (TILE_W + 6), tx = i % (TILE_W + 6);
        s_in[ty][tx] = src[(size_t)reflect101(y0 + ty - 3, h) * w + reflect101(x0 + tx - 3, w)];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (TILE_H + 6) * TILE_W; i += THREADS) {
        const int ty = i / TILE_W, tx = i % TILE_W;
        float acc = 0.f;
        if (x0 + tx < w / 32 * 32) {   // OpenCV's row filter fuses in its 32-pixel vector steps, not in its scalar tail
#pragma unroll
            for (int j = 0; j < 7; ++j) acc = __fmaf_rn(L.taps[j], (float)s_in[ty][tx + j], acc);
        } else {
#pragma unroll
            for (int j = 0; j < 7; ++j) acc = __fadd_rn(acc, __fmul_rn(L.taps[j], (float)s_in[ty][tx + j]));
        }
        s_row[ty][tx] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TILE_H * TILE_W; i += THREADS) {
        const int ty = i / TILE_W, tx = i % TILE_W, x = x0 + tx, y = y0 + ty;
        if (x >= w || y >= h) continue;
        float acc = __fmul_rn(L.taps[3], s_row[ty + 3][tx]);
#pragma unroll
        for (int k = 1; k <= 3; ++k) acc = __fmaf_rn(L.taps[3 + k], __fadd_rn(s_row[ty + 3 + k][tx], s_row[ty + 3 - k][tx]), acc);
        const int v = __float2int_rn(acc);
        dst[(size_t)y * w + x] = (uint8_t)min(max(v, 0), 255);
    }
}

// border filter, one CTA per image: an ordered block scan compacts the survivors to rows kp_off[i] + k
__global__ void __launch_bounds__(THREADS)
orb_filter_kernel(int W, int H, int edge, const int32_t* __restrict__ kp_off, const float* __restrict__ kp_xy,
                  int32_t* src_idx, int32_t* counts) {
    __shared__ int s_warp[THREADS / 32], s_base;
    const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int a0 = kp_off[img], n = kp_off[img + 1] - a0;
    const bool any = W > 2 * edge && H > 2 * edge;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int base = 0; base < n; base += THREADS) {
        const int j = base + tid;
        int keep = 0;
        if (j < n && any) {
            const int rx = __float2int_rn(kp_xy[2 * (size_t)(a0 + j)]), ry = __float2int_rn(kp_xy[2 * (size_t)(a0 + j) + 1]);
            keep = rx >= edge && rx < W - edge && ry >= edge && ry < H - edge;
        }
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = 0, tot = 0;
        for (int q = 0; q < THREADS / 32; ++q) {
            if (q < warp) before += s_warp[q];
            tot += s_warp[q];
        }
        if (keep) src_idx[a0 + s_base + before + __popc(bal & ((1u << lane) - 1u))] = j;
        __syncthreads();
        if (tid == 0) s_base += tot;
        __syncthreads();
    }
    if (tid == 0) counts[img] = s_base;
}

__global__ void __launch_bounds__(THREADS)
orb_describe_kernel(OrbDevLevels L, int n_img, const uint8_t* __restrict__ images, const uint8_t* __restrict__ raw_pyr,
                    const uint8_t* __restrict__ blur_pyr, const int32_t* __restrict__ kp_off, const float* __restrict__ kp_xy,
                    const int32_t* __restrict__ kp_oct, const float* __restrict__ kp_angle, const int32_t* __restrict__ src_idx,
                    const int32_t* __restrict__ counts, float* out_angle, uint8_t* out_desc) {
    const int lane = threadIdx.x & 31;
    const int row = (int)((blockIdx.x * (size_t)THREADS + threadIdx.x) >> 5);
    if (row >= kp_off[n_img]) return;
    int lo = 0, hi = n_img;   // image of this row: the last i with kp_off[i] <= row
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (kp_off[mid] <= row) lo = mid; else hi = mid;
    }
    const int img = lo, a0 = kp_off[img];
    if (row - a0 >= counts[img]) return;
    const int k = a0 + src_idx[row];
    const int l = kp_oct[k], w = L.w[l], h = L.h[l];
    const uint8_t* raw = raw_level(L, images, raw_pyr, img, l);
    const uint8_t* blur = blur_pyr + (size_t)img * L.blur_stride + L.blur_off[l];
    const int cx = __float2int_rn(__fmul_rn(kp_xy[2 * (size_t)k], L.inv[l]));
    const int cy = __float2int_rn(__fmul_rn(kp_xy[2 * (size_t)k + 1], L.inv[l]));
    float angle;
    if (kp_angle) {
        angle = kp_angle[k];
    } else {   // intensity centroid over the radius-15 disc: lane u + 15 sums column u; integer sums, so any order
        const int u = lane - 15;
        int m10 = 0, m01 = 0;
        if (lane < 31) {
            const int au = abs(u);
            for (int v = -15; v <= 15; ++v) {
                if (au > c_umax[abs(v)]) continue;
                const int x = cx + u, y = cy + v;
                const int p = (x >= 0 && x < w && y >= 0 && y < h) ? raw[(size_t)y * w + x]
                                                                   : raw[(size_t)reflect101(y, h) * w + reflect101(x, w)];
                m10 += u * p;
                m01 += v * p;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            m10 += __shfl_xor_sync(0xFFFFFFFFu, m10, o);
            m01 += __shfl_xor_sync(0xFFFFFFFFu, m01, o);
        }
        angle = fast_atan2((float)m01, (float)m10);
    }
    double sd, cd;
    sincos((double)__fmul_rn(angle, 0.0174532924f), &sd, &cd);   // (float)(CV_PI / 180.f)
    const float a = (float)cd, b = (float)sd;
    uint32_t word[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {   // bit 32 q + lane
        const signed char* pp = c_pattern[32 * q + lane];
        int v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float fx = (float)pp[2 * e], fy = (float)pp[2 * e + 1];
            const int x = cx + __float2int_rn(__fsub_rn(__fmul_rn(fx, a), __fmul_rn(fy, b)));
            const int y = cy + __float2int_rn(__fadd_rn(__fmul_rn(fx, b), __fmul_rn(fy, a)));
            v[e] = (x >= 0 && x < w && y >= 0 && y < h) ? blur[(size_t)y * w + x]
                                                        : raw[(size_t)reflect101(y, h) * w + reflect101(x, w)];
        }
        word[q] = __ballot_sync(0xFFFFFFFFu, v[0] < v[1]);
    }
    if (lane < 8) {
        uint32_t wv = word[0];
#pragma unroll
        for (int q = 1; q < 8; ++q)
            if (lane == q) wv = word[q];
        reinterpret_cast<uint32_t*>(out_desc + 32 * (size_t)row)[lane] = wv;
    }
    if (lane == 0) out_angle[row] = angle;
}

// ---- key-point selection (computeKeyPoints): FAST-9/16 + NMS, border filter, retainBest, Harris ----

// exclusive scan of one value per thread over the CTA; *total gets the CTA's sum
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    int before = 0, tot = 0;
    for (int q = 0; q < THREADS / 32; ++q) {
        if (q < warp) before += s_warp[q];
        tot += s_warp[q];
    }
    __syncthreads();
    *total = tot;
    return before + inc - v;
}

// FAST score: the largest t for which 9 contiguous circle pixels all differ from the centre by more than t in one direction,
// i.e. max over the 16 arcs of (min signed difference) - 1, bright (ring - centre) or dark (centre - ring).  The circle of
// radius 3 is listed contiguously, as OpenCV's makeOffsets lists it.
__device__ __forceinline__ int fast_score(const uint8_t (*s)[TILE_W + 8], int cy, int cx) {
    constexpr int DX[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    constexpr int DY[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    const int c = s[cy][cx];
    int d[16], mn[16], mx[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) d[k] = (int)s[cy + DY[k]][cx + DX[k]] - c;
#pragma unroll
    for (int k = 0; k < 16; ++k) { mn[k] = min(d[k], d[(k + 1) & 15]); mx[k] = max(d[k], d[(k + 1) & 15]); }   // arcs of 2
    int mn4[16], mx4[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) { mn4[k] = min(mn[k], mn[(k + 2) & 15]); mx4[k] = max(mx[k], mx[(k + 2) & 15]); }   // of 4
    int bright = -512, dark = 512;
#pragma unroll
    for (int k = 0; k < 16; ++k) {   // arcs of 9: 8 + the next pixel
        bright = max(bright, min(min(mn4[k], mn4[(k + 4) & 15]), d[(k + 8) & 15]));
        dark = min(dark, max(max(mx4[k], mx4[(k + 4) & 15]), d[(k + 8) & 15]));
    }
    return max(bright, -dark) - 1;
}

// one level: score (FAST corners only), 3x3 non-max suppression with non-corners as 0, the level's border filter; writes the
// u8 score map (0: not kept; a kept corner scores >= 1) and adds the kept scores' histogram of (image, level) to hist
__global__ void __launch_bounds__(THREADS)
orb_fast_kernel(OrbDevLevels L, OrbDetectLevels D, int l, const uint8_t* __restrict__ images, const uint8_t* __restrict__ raw_pyr,
                const int32_t* __restrict__ fast_th, uint8_t* score, uint32_t* hist) {
    __shared__ uint8_t s_in[TILE_H + 8][TILE_W + 8];    // tile + 3-pixel circle + 1-pixel NMS ring
    __shared__ uint8_t s_sc[TILE_H + 2][TILE_W + 2];
    __shared__ uint32_t s_hist[256];
    const int img = blockIdx.z, w = L.w[l], h = L.h[l], tid = threadIdx.x;
    const uint8_t* src = raw_level(L, images, raw_pyr, img, l);
    const int x0 = blockIdx.x * TILE_W, y0 = blockIdx.y * TILE_H;
    for (int i = tid; i < 256; i += THREADS) s_hist[i] = 0;
    for (int i = tid; i < (TILE_H + 8) * (TILE_W + 8); i += THREADS) {
        const int ty = i / (TILE_W + 8), tx = i % (TILE_W + 8), y = y0 + ty - 4, x = x0 + tx - 4;
        s_in[ty][tx] = (x >= 0 && x < w && y >= 0 && y < h) ? src[(size_t)y * w + x] : 0;
    }
    __syncthreads();
    const int th = fast_th[img];
    for (int i = tid; i < (TILE_H + 2) * (TILE_W + 2); i += THREADS) {
        const int ty = i / (TILE_W + 2), tx = i % (TILE_W + 2), y = y0 + ty - 1, x = x0 + tx - 1;
        int sc = 0;
        if (x >= 3 && x < w - 3 && y >= 3 && y < h - 3) {
            sc = fast_score(s_in, ty + 3, tx + 3);
            if (sc < th) sc = 0;
        }
        s_sc[ty][tx] = (uint8_t)sc;
    }
    __syncthreads();
    uint8_t* dst = score + (size_t)img * L.blur_stride + L.blur_off[l];
    for (int i = tid; i < TILE_H * TILE_W; i += THREADS) {
        const int ty = i / TILE_W, tx = i % TILE_W, x = x0 + tx, y = y0 + ty;
        if (x >= w || y >= h) continue;
        const int v = s_sc[ty + 1][tx + 1];
        bool keep = v > 0 && x >= D.edge && x < w - D.edge && y >= D.edge && y < h - D.edge;
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx)
                if (dy != 1 || dx != 1) keep = keep && v > s_sc[ty + dy][tx + dx];
        dst[(size_t)y * w + x] = keep ? (uint8_t)v : 0;
        if (keep) atomicAdd(&s_hist[v], 1u);
    }
    __syncthreads();
    uint32_t* gh = hist + ((size_t)img * L.n + l) * 256;
    for (int i = tid; i < 256; i += THREADS)
        if (s_hist[i]) atomicAdd(&gh[i], s_hist[i]);
}

// retainBest on the FAST score of (image, level): keep every point scoring >= the keep1-th largest score, which is the largest
// v with count(score >= v) >= keep1.  cut 1: keep all; 256: keep none (retainBest(0))
__global__ void orb_fast_cut_kernel(int n, OrbDetectLevels D, int nl, const uint32_t* __restrict__ hist, int32_t* cut) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * nl) return;
    const int keep = D.keep1[i % nl];
    const uint32_t* hh = hist + 256 * (size_t)i;
    int c = 256;
    if (keep > 0) {
        uint32_t acc = 0;
        c = 1;
        for (int v = 255; v >= 1; --v) {
            acc += hh[v];
            if (acc >= (uint32_t)keep) { c = v; break; }
        }
    }
    cut[i] = c;
}

__device__ __forceinline__ int row_level(const OrbDetectLevels& D, int nl, int r) {
    int l = 0;
    while (l + 1 < nl && r >= D.row0[l + 1]) ++l;
    return l;
}

// one warp per row of the stacked levels: write == false counts the row's selected points into row_cnt; write == true
// writes them at sel_off[img] + row_base[row] + rank within the row (x ascending)
template <bool WRITE>
__global__ void __launch_bounds__(THREADS)
orb_fast_rows_kernel(OrbDevLevels L, OrbDetectLevels D, const uint8_t* __restrict__ score, const int32_t* __restrict__ cut,
                     int32_t* row_cnt, const int32_t* __restrict__ row_base, const int32_t* __restrict__ sel_off, int2* lxy,
                     float* xy, int32_t* oct, float* resp, int32_t* rank) {
    const int img = blockIdx.y, R = D.row0[L.n], lane = threadIdx.x & 31;
    const int r = blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5);
    if (r >= R) return;
    const int l = row_level(D, L.n, r), y = r - D.row0[l], w = L.w[l];
    const uint8_t* row = score + (size_t)img * L.blur_stride + L.blur_off[l] + (size_t)y * w;
    const int c = cut[img * L.n + l];
    int n = 0;
    const int a0 = WRITE ? sel_off[img] : 0, base = WRITE ? row_base[(size_t)img * (R + 1) + r] : 0;
    const float ls = D.layer_scale[l];
    if (y >= D.edge && y < L.h[l] - D.edge) {
        for (int xb = D.edge; xb < w - D.edge; xb += 32) {
            const int x = xb + lane;
            const int v = x < w - D.edge ? row[x] : 0;
            const bool keep = v >= c;
            const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
            if (WRITE && keep) {
                const int q = base + n + __popc(bal & ((1u << lane) - 1u)), k = a0 + q;
                lxy[k] = make_int2(x, y);
                xy[2 * (size_t)k] = __fmul_rn((float)x, ls);
                xy[2 * (size_t)k + 1] = __fmul_rn((float)y, ls);
                oct[k] = l;
                resp[k] = (float)v;
                rank[k] = q;
            }
            n += __popc(bal);
        }
    }
    if (!WRITE && lane == 0) row_cnt[(size_t)img * R + r] = n;
}

// one CTA per image: row_base[img][0..R] = exclusive scan of the row counts; img_cnt[img] = the image's total
__global__ void __launch_bounds__(THREADS)
orb_row_scan_kernel(int R, const int32_t* __restrict__ row_cnt, int32_t* row_base, int32_t* img_cnt) {
    __shared__ int s_warp[THREADS / 32];
    const int img = blockIdx.x;
    int carry = 0;
    for (int b = 0; b <= R; b += THREADS) {
        const int r = b + threadIdx.x;
        const int v = r < R ? row_cnt[(size_t)img * R + r] : 0;
        int tot;
        const int ex = block_exclusive_scan(v, s_warp, &tot);
        if (r <= R) row_base[(size_t)img * (R + 1) + r] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) img_cnt[img] = carry;
}

// one CTA: off[0..n] = exclusive scan over images of the sums of per consecutive values of v; cnt[i] (optional) = the sums
__global__ void __launch_bounds__(THREADS)
orb_offsets_kernel(int n, const int32_t* __restrict__ v, int per, int32_t* off, int32_t* cnt) {
    __shared__ int s_warp[THREADS / 32];
    int carry = 0;
    for (int b = 0; b < n; b += THREADS) {
        const int i = b + threadIdx.x;
        int c = 0;
        if (i < n) {
            for (int q = 0; q < per; ++q) c += v[(size_t)i * per + q];
            if (cnt) cnt[i] = c;
        }
        int tot;
        const int ex = block_exclusive_scan(c, s_warp, &tot);
        if (i < n) off[i] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) off[n] = carry;
}

__device__ __forceinline__ int image_of_row(const int32_t* off, int n_img, int row) {   // the last i with off[i] <= row
    int lo = 0, hi = n_img;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= row) lo = mid; else hi = mid;
    }
    return lo;
}

// Harris response of one candidate on its raw level (OpenCV's HarrisResponses, block 7, k 0.04): integer sums of the
// Sobel-like gradients over the 7x7 block, then the response in float, unfused, in OpenCV's order.  Outside the level the
// pixels are the level's BORDER_REFLECT_101 (OpenCV's pyramid border), reached only with edge_threshold < 4.
__global__ void __launch_bounds__(THREADS)
orb_harris_kernel(OrbDevLevels L, OrbDetectLevels D, int n_img, int n_cand, const uint8_t* __restrict__ images,
                  const uint8_t* __restrict__ raw_pyr, const int32_t* __restrict__ sel_off, const int2* __restrict__ lxy,
                  const int32_t* __restrict__ oct, float* hresp) {
    const int k = blockIdx.x * THREADS + threadIdx.x;
    if (k >= n_cand) return;
    const int img = image_of_row(sel_off, n_img, k), l = oct[k], w = L.w[l], h = L.h[l];
    const uint8_t* raw = raw_level(L, images, raw_pyr, img, l);
    const int2 c = lxy[k];
    int p[9][9];
    const bool inside = c.x >= 4 && c.x < w - 4 && c.y >= 4 && c.y < h - 4;
#pragma unroll
    for (int i = 0; i < 9; ++i)
#pragma unroll
        for (int j = 0; j < 9; ++j) {
            const int y = c.y - 4 + i, x = c.x - 4 + j;
            p[i][j] = inside ? raw[(size_t)y * w + x] : raw[(size_t)reflect101(y, h) * w + reflect101(x, w)];
        }
    int a = 0, b = 0, cc = 0;
#pragma unroll
    for (int i = 1; i < 8; ++i)
#pragma unroll
        for (int j = 1; j < 8; ++j) {
            const int ix = (p[i][j + 1] - p[i][j - 1]) * 2 + (p[i - 1][j + 1] - p[i - 1][j - 1]) + (p[i + 1][j + 1] - p[i + 1][j - 1]);
            const int iy = (p[i + 1][j] - p[i - 1][j]) * 2 + (p[i + 1][j - 1] - p[i - 1][j - 1]) + (p[i + 1][j + 1] - p[i - 1][j + 1]);
            a += ix * ix;
            b += iy * iy;
            cc += ix * iy;
        }
    const float fa = __int2float_rn(a), fb = __int2float_rn(b), fc = __int2float_rn(cc), s = __fadd_rn(fa, fb);
    const float r = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, s), s));
    hresp[k] = __fmul_rn(r, D.harris_scale4);
}

// order-preserving key of a float response (+0 and -0 compare equal, as retainBest's float comparison has them)
__device__ __forceinline__ uint32_t response_key(float f) {
    const uint32_t u = f == 0.f ? 0u : __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// retainBest on the Harris response, one CTA per (image, level): the keep2-th largest key by an 8-bit radix select (the
// pattern of solve.cu's block_select_wide); cut_key = that key (0: keep all), lvl_keep = how many keys are >= it
__global__ void __launch_bounds__(THREADS)
orb_harris_cut_kernel(OrbDevLevels L, OrbDetectLevels D, const int32_t* __restrict__ row_base, const int32_t* __restrict__ sel_off,
                      const float* __restrict__ hresp, uint32_t* cut_key, int32_t* lvl_keep) {
    __shared__ uint32_t s_hist[256];
    __shared__ uint32_t s_prefix, s_eq;
    __shared__ int s_k;
    const int img = blockIdx.x / L.n, l = blockIdx.x % L.n, R = D.row0[L.n], tid = threadIdx.x;
    const int32_t* rb = row_base + (size_t)img * (R + 1);
    const int a0 = sel_off[img] + rb[D.row0[l]], m = rb[D.row0[l + 1]] - rb[D.row0[l]], k = D.keep2[l];
    if (k <= 0 || m <= k) {
        if (tid == 0) { cut_key[blockIdx.x] = 0u; lvl_keep[blockIdx.x] = k <= 0 ? 0 : m; }
        return;
    }
    uint32_t prefix = 0u;
    int kk = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
        const uint32_t hmask = shift == 24 ? 0u : (0xFFFFFFFFu << (shift + 8));
        for (int i = tid; i < 256; i += THREADS) s_hist[i] = 0u;
        __syncthreads();
        for (int i = tid; i < m; i += THREADS) {
            const uint32_t key = response_key(hresp[a0 + i]);
            if ((key & hmask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {   // the digit that holds rank kk, counting from the top
            uint32_t acc = 0;
            int d = 255;
            for (; d > 0; --d) {
                if (acc + s_hist[d] >= (uint32_t)kk) break;
                acc += s_hist[d];
            }
            s_prefix = prefix | ((uint32_t)d << shift);
            s_k = kk - (int)acc;
            s_eq = s_hist[d];
        }
        __syncthreads();
        prefix = s_prefix;
        kk = s_k;
    }
    if (tid == 0) {   // keys above the cut: k - kk; keys equal to it: the last digit's bin
        cut_key[blockIdx.x] = prefix;
        lvl_keep[blockIdx.x] = k - kk + (int)s_eq;
    }
}

// one CTA per image: the candidates whose Harris key is >= their level's cut, in candidate order, densely at out_off[img] + rank
__global__ void __launch_bounds__(THREADS)
orb_harris_write_kernel(OrbDetectLevels D, int nl, const int32_t* __restrict__ sel_off, const float* __restrict__ xy,
                        const int32_t* __restrict__ oct, const float* __restrict__ hresp, const uint32_t* __restrict__ cut_key,
                        const int32_t* __restrict__ out_off, float* out_xy, int32_t* out_oct, float* out_resp, int32_t* out_rank) {
    __shared__ int s_warp[THREADS / 32];
    const int img = blockIdx.x, a0 = sel_off[img], n = sel_off[img + 1] - a0, o0 = out_off[img];
    int base = 0;
    for (int b = 0; b < n; b += THREADS) {
        const int j = b + threadIdx.x, k = a0 + j;
        int keep = 0, l = 0;
        if (j < n) {
            l = oct[k];
            keep = D.keep2[l] > 0 && response_key(hresp[k]) >= cut_key[img * nl + l];
        }
        int tot;
        const int ex = block_exclusive_scan(keep, s_warp, &tot);
        if (keep) {
            const int q = base + ex, o = o0 + q;
            out_xy[2 * (size_t)o] = xy[2 * (size_t)k];
            out_xy[2 * (size_t)o + 1] = xy[2 * (size_t)k + 1];
            out_oct[o] = l;
            out_resp[o] = hresp[k];
            out_rank[o] = q;
        }
        base += tot;
    }
}

}  // namespace orb

using namespace orb;

cudaError_t orb_upload_tables() {
    int umax[16];
    {   // ORB's umax for half patch 15
        const int half = 15;
        const int vmax = (int)floor(half * sqrt(2.f) / 2 + 1), vmin = (int)ceil(half * sqrt(2.f) / 2);
        int u[17];
        for (int v = 0; v <= vmax; ++v) u[v] = (int)lrint(sqrt((double)half * half - v * v));
        for (int v = half, v0 = 0; v >= vmin; --v) {
            while (u[v0] == u[v0 + 1]) ++v0;
            u[v] = v0;
            ++v0;
        }
        for (int v = 0; v < 16; ++v) umax[v] = u[v];
    }
    cudaError_t e = cudaMemcpyToSymbol(c_umax, umax, sizeof(umax));
    if (e != cudaSuccess) return e;
    return cudaMemcpyToSymbol(c_pattern, kOrbPattern31, sizeof(kOrbPattern31));
}

void launch_orb_pyramid(const OrbDevLevels& L, int n_img, const uint8_t* images, uint8_t* raw_pyr, uint8_t* blur_pyr,
                        const int32_t* const* rs_tab, cudaStream_t s, int* launches) {
    for (int l = 0; l < L.n; ++l) {
        const dim3 grid((L.w[l] + TILE_W - 1) / TILE_W, (L.h[l] + TILE_H - 1) / TILE_H, n_img);
        if (l > 0) {
            orb_resize_kernel<<<grid, THREADS, 0, s>>>(L, l, images, raw_pyr, rs_tab[2 * l], rs_tab[2 * l + 1]);
            ++*launches;
        }
        orb_blur_kernel<<<grid, THREADS, 0, s>>>(L, l, images, raw_pyr, blur_pyr);
        ++*launches;
    }
}

void launch_orb_describe(const OrbDevLevels& L, int n_img, const uint8_t* images, const uint8_t* raw_pyr,
                         const uint8_t* blur_pyr, const int32_t* kp_off, int n_rows, const float* kp_xy, const int32_t* kp_oct,
                         const float* kp_angle, const int32_t* src_idx, const int32_t* counts, float* out_angle,
                         uint8_t* out_desc, cudaStream_t s, int* launches) {
    if (n_rows <= 0) return;
    const int blocks = (int)(((size_t)n_rows * 32 + THREADS - 1) / THREADS);
    orb_describe_kernel<<<blocks, THREADS, 0, s>>>(L, n_img, images, raw_pyr, blur_pyr, kp_off, kp_xy, kp_oct, kp_angle,
                                                   src_idx, counts, out_angle, out_desc);
    ++*launches;
}

cudaError_t launch_orb(const OrbDevLevels& L, int n_img, int W, int H, int edge, const uint8_t* images, uint8_t* raw_pyr,
                       uint8_t* blur_pyr, const int32_t* const* rs_tab, const int32_t* kp_off, int n_rows, const float* kp_xy,
                       const int32_t* kp_oct, const float* kp_angle, int32_t* src_idx, int32_t* counts, float* out_angle,
                       uint8_t* out_desc, cudaStream_t s, cudaEvent_t* ev, int* launches) {
    if (n_img <= 0) return cudaSuccess;
    // ev (optional): [0] before the pyramid, [1] after it and the blur, [2] after the filter, [3] after the descriptors
    if (ev) cudaEventRecord(ev[0], s);
    launch_orb_pyramid(L, n_img, images, raw_pyr, blur_pyr, rs_tab, s, launches);
    if (ev) cudaEventRecord(ev[1], s);
    orb_filter_kernel<<<n_img, THREADS, 0, s>>>(W, H, edge, kp_off, kp_xy, src_idx, counts);
    ++*launches;
    if (ev) cudaEventRecord(ev[2], s);
    launch_orb_describe(L, n_img, images, raw_pyr, blur_pyr, kp_off, n_rows, kp_xy, kp_oct, kp_angle, src_idx, counts,
                        out_angle, out_desc, s, launches);
    if (ev) cudaEventRecord(ev[3], s);
    return cudaGetLastError();
}

void launch_orb_fast_select(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, const uint8_t* images,
                            const uint8_t* raw_pyr, const int32_t* fast_th, uint8_t* score, uint32_t* hist, int32_t* cut,
                            int32_t* row_cnt, int32_t* row_base, int32_t* img_cnt, int32_t* sel_off, cudaStream_t s,
                            cudaEvent_t ev_fast_done, int* launches) {
    cudaMemsetAsync(hist, 0, (size_t)n_img * L.n * 256 * sizeof(uint32_t), s);
    for (int l = 0; l < L.n; ++l) {
        const dim3 grid((L.w[l] + TILE_W - 1) / TILE_W, (L.h[l] + TILE_H - 1) / TILE_H, n_img);
        orb_fast_kernel<<<grid, THREADS, 0, s>>>(L, D, l, images, raw_pyr, fast_th, score, hist);
        ++*launches;
    }
    if (ev_fast_done) cudaEventRecord(ev_fast_done, s);
    orb_fast_cut_kernel<<<(n_img * L.n + THREADS - 1) / THREADS, THREADS, 0, s>>>(n_img, D, L.n, hist, cut);
    const int R = D.row0[L.n];
    const dim3 rows((R + THREADS / 32 - 1) / (THREADS / 32), n_img);
    orb_fast_rows_kernel<false><<<rows, THREADS, 0, s>>>(L, D, score, cut, row_cnt, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                         nullptr, nullptr);
    orb_row_scan_kernel<<<n_img, THREADS, 0, s>>>(R, row_cnt, row_base, img_cnt);
    orb_offsets_kernel<<<1, THREADS, 0, s>>>(n_img, img_cnt, 1, sel_off, nullptr);
    *launches += 4;
}

void launch_orb_fast_write(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, const uint8_t* score, const int32_t* cut,
                           const int32_t* row_base, const int32_t* sel_off, int2* lxy, float* xy, int32_t* oct, float* resp,
                           int32_t* rank, cudaStream_t s, int* launches) {
    const int R = D.row0[L.n];
    const dim3 rows((R + THREADS / 32 - 1) / (THREADS / 32), n_img);
    orb_fast_rows_kernel<true><<<rows, THREADS, 0, s>>>(L, D, score, cut, nullptr, row_base, sel_off, lxy, xy, oct, resp, rank);
    ++*launches;
}

void launch_orb_harris_select(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, int n_cand, const uint8_t* images,
                              const uint8_t* raw_pyr, const int32_t* row_base, const int32_t* sel_off, const int2* lxy,
                              const int32_t* oct, float* hresp, uint32_t* cut_key, int32_t* lvl_keep, int32_t* out_off,
                              int32_t* out_cnt, cudaStream_t s, int* launches) {
    if (n_cand > 0) {
        orb_harris_kernel<<<(n_cand + THREADS - 1) / THREADS, THREADS, 0, s>>>(L, D, n_img, n_cand, images, raw_pyr, sel_off,
                                                                               lxy, oct, hresp);
        ++*launches;
    }
    orb_harris_cut_kernel<<<n_img * L.n, THREADS, 0, s>>>(L, D, row_base, sel_off, hresp, cut_key, lvl_keep);
    orb_offsets_kernel<<<1, THREADS, 0, s>>>(n_img, lvl_keep, L.n, out_off, out_cnt);
    *launches += 2;
}

void launch_orb_harris_write(const OrbDevLevels& L, const OrbDetectLevels& D, int n_img, const int32_t* sel_off,
                             const float* xy, const int32_t* oct, const float* hresp, const uint32_t* cut_key,
                             const int32_t* out_off, float* out_xy, int32_t* out_oct, float* out_resp, int32_t* out_rank,
                             cudaStream_t s, int* launches) {
    orb_harris_write_kernel<<<n_img, THREADS, 0, s>>>(D, L.n, sel_off, xy, oct, hresp, cut_key, out_off, out_xy, out_oct,
                                                      out_resp, out_rank);
    ++*launches;
}

}  // namespace plstvo
