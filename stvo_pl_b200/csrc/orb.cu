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

cudaError_t launch_orb(const OrbDevLevels& L, int n_img, int W, int H, int edge, const uint8_t* images, uint8_t* raw_pyr,
                       uint8_t* blur_pyr, const int32_t* const* rs_tab, const int32_t* kp_off, int n_rows, const float* kp_xy,
                       const int32_t* kp_oct, const float* kp_angle, int32_t* src_idx, int32_t* counts, float* out_angle,
                       uint8_t* out_desc, cudaStream_t s, cudaEvent_t* ev, int* launches) {
    if (n_img <= 0) return cudaSuccess;
    // ev (optional): [0] before the pyramid, [1] after it and the blur, [2] after the filter, [3] after the descriptors
    if (ev) cudaEventRecord(ev[0], s);
    for (int l = 0; l < L.n; ++l) {
        const dim3 grid((L.w[l] + TILE_W - 1) / TILE_W, (L.h[l] + TILE_H - 1) / TILE_H, n_img);
        if (l > 0) {
            orb_resize_kernel<<<grid, THREADS, 0, s>>>(L, l, images, raw_pyr, rs_tab[2 * l], rs_tab[2 * l + 1]);
            ++*launches;
        }
        orb_blur_kernel<<<grid, THREADS, 0, s>>>(L, l, images, raw_pyr, blur_pyr);
        ++*launches;
    }
    if (ev) cudaEventRecord(ev[1], s);
    orb_filter_kernel<<<n_img, THREADS, 0, s>>>(W, H, edge, kp_off, kp_xy, src_idx, counts);
    ++*launches;
    if (ev) cudaEventRecord(ev[2], s);
    if (n_rows > 0) {
        const int blocks = (int)(((size_t)n_rows * 32 + THREADS - 1) / THREADS);
        orb_describe_kernel<<<blocks, THREADS, 0, s>>>(L, n_img, images, raw_pyr, blur_pyr, kp_off, kp_xy, kp_oct, kp_angle,
                                                       src_idx, counts, out_angle, out_desc);
        ++*launches;
    }
    if (ev) cudaEventRecord(ev[3], s);
    return cudaGetLastError();
}

}  // namespace plstvo
