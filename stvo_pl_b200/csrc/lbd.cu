// lbd.cu — LBD line descriptors of given octave-0 key lines (BinaryDescriptor::compute with default Params,
// 3rdparty/line_descriptor/src/binary_descriptor_custom.cpp), bit-exact with the reference evaluated unfused.
//
//   lbd_grad_kernel      per image: OpenCV's fixed-point GaussianBlur(5x5, sigma 1) of the 8-bit image, then Sobel 3x3
//                        (CV_16S) of the blurred image, both BORDER_REFLECT_101, into one short2 (dx, dy) per pixel
//   lbd_describe_kernel  per key line (64 threads): the 63 rows of the line support region, the 9 band statistics,
//                        normalisation, clamp at 0.4 and the 32 bytes of binaryConversion
//
// Every float operation is spelled with an _rn intrinsic in the reference's source order: nvcc would otherwise contract
// a * b + c into an FMA, which the reference (built -ffp-contract=off) does not do.  The line direction dL = (cos, sin) of
// the float angle comes in precomputed: the reference's cos(float) / sin(float) are the C library's cosf / sinf, which the
// host evaluates (capi.cu), since CUDA's cosf / sinf do not round the same way.
#include "common.cuh"

namespace plstvo {
namespace {

constexpr int LBD_TILE_W = 64, LBD_TILE_H = 16;
constexpr int LBD_SRC_W = LBD_TILE_W + 6, LBD_SRC_H = LBD_TILE_H + 6;   // 2 px blur halo + 1 px Sobel halo, each side
constexpr int LBD_BLR_W = LBD_TILE_W + 2, LBD_BLR_H = LBD_TILE_H + 2;
constexpr int LBD_BANDS = 9, LBD_BAND_W = 7, LBD_ROWS = LBD_BANDS * LBD_BAND_W, LBD_HALF_H = (LBD_ROWS - 1) / 2;
constexpr int LBD_DESC = LBD_BANDS * 8;

// createGaussianKernelBitExact(sigma 1, 5 taps) for 8-bit images: 8 fractional bits
__constant__ int c_blur_taps[5] = {14, 62, 104, 62, 14};
__constant__ float c_coef_g[LBD_ROWS];       // (float)gaussCoefG_[h]
__constant__ float c_coef_l[3 * LBD_BAND_W]; // (float)gaussCoefL_[i]
__constant__ signed char c_comb[32][2] = {
    {0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {0, 6}, {1, 2}, {1, 3}, {1, 4}, {1, 5}, {1, 6}, {2, 3}, {2, 4}, {2, 5}, {2, 6}, {2, 7},
    {2, 8}, {3, 4}, {3, 5}, {3, 6}, {3, 7}, {3, 8}, {4, 5}, {4, 6}, {4, 7}, {4, 8}, {5, 6}, {5, 7}, {5, 8}, {6, 7}, {6, 8}, {7, 8}};

// cv::borderInterpolate(p, len, BORDER_REFLECT_101), iterated as OpenCV does for images narrower than the kernel
__device__ __forceinline__ int reflect101(int p, int len) {
    if (len == 1) return 0;
    while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

// grid (tiles x, tiles y, image); 256 threads.  Reflect-101 is applied twice: to the source for the blur and to the
// blurred image for the Sobel, so a blurred halo cell outside the image holds the blurred value of its reflected pixel.
__global__ void __launch_bounds__(256) lbd_grad_kernel(const uint8_t* __restrict__ images, int W, int H, int img0,
                                                       const int32_t* __restrict__ kl_off, short2* __restrict__ grad) {
    const int img = img0 + (int)blockIdx.z;
    if (kl_off[img + 1] == kl_off[img]) return;   // no lines: the gradient is never read
    __shared__ uint8_t s_src[LBD_SRC_H][LBD_SRC_W];     // source at reflect101(y0 - 3 + r), reflect101(x0 - 3 + c)
    __shared__ uint32_t s_row[LBD_SRC_H][LBD_BLR_W];    // horizontal pass (8.8 fixed point) at the blurred tile's columns
    __shared__ int16_t s_blur[LBD_BLR_H][LBD_BLR_W];    // blurred value at reflect101(y0 - 1 + r), reflect101(x0 - 1 + c)
    const int x0 = blockIdx.x * LBD_TILE_W, y0 = blockIdx.y * LBD_TILE_H, t = threadIdx.x;
    const uint8_t* src = images + (size_t)img * W * H;
    for (int i = t; i < LBD_SRC_H * LBD_SRC_W; i += blockDim.x) {
        const int r = i / LBD_SRC_W, c = i % LBD_SRC_W;
        s_src[r][c] = src[(size_t)reflect101(y0 - 3 + r, H) * W + reflect101(x0 - 3 + c, W)];
    }
    __syncthreads();
    // blurred cell c stands for image column p = x0 - 1 + c; only p in [-1, W] is ever read by the Sobel.  Its value is the
    // blur at q = reflect101(p), whose taps q - 2 .. q + 2 sit at s_src columns q - x0 + 1 .. q - x0 + 5.
    for (int i = t; i < LBD_SRC_H * LBD_BLR_W; i += blockDim.x) {
        const int r = i / LBD_BLR_W, c = i % LBD_BLR_W, p = x0 - 1 + c;
        uint32_t a = 0;
        if (p >= -1 && p <= W) {
            const int q = reflect101(p, W) - x0 + 1;
#pragma unroll
            for (int k = 0; k < 5; ++k) a += (uint32_t)c_blur_taps[k] * s_src[r][q + k];
        }
        s_row[r][c] = a;
    }
    __syncthreads();
    for (int i = t; i < LBD_BLR_H * LBD_BLR_W; i += blockDim.x) {
        const int r = i / LBD_BLR_W, c = i % LBD_BLR_W, p = y0 - 1 + r;
        int v = 0;
        if (p >= -1 && p <= H) {
            const int q = reflect101(p, H) - y0 + 1;
            uint32_t a = 0;
#pragma unroll
            for (int k = 0; k < 5; ++k) a += (uint32_t)c_blur_taps[k] * s_row[q + k][c];
            v = (int)min((a + (1u << 15)) >> 16, 255u);
        }
        s_blur[r][c] = (int16_t)v;
    }
    __syncthreads();
    short2* out = grad + (size_t)img * W * H;
    for (int i = t; i < LBD_TILE_H * LBD_TILE_W; i += blockDim.x) {
        const int r = i / LBD_TILE_W, c = i % LBD_TILE_W, x = x0 + c, y = y0 + r;
        if (x >= W || y >= H) continue;
        const int R = r + 1, Cc = c + 1;
        const int dx = (s_blur[R - 1][Cc + 1] - s_blur[R - 1][Cc - 1]) + 2 * (s_blur[R][Cc + 1] - s_blur[R][Cc - 1]) +
                       (s_blur[R + 1][Cc + 1] - s_blur[R + 1][Cc - 1]);
        const int dy = (s_blur[R + 1][Cc - 1] - s_blur[R - 1][Cc - 1]) + 2 * (s_blur[R + 1][Cc] - s_blur[R - 1][Cc]) +
                       (s_blur[R + 1][Cc + 1] - s_blur[R - 1][Cc + 1]);
        out[(size_t)y * W + x] = make_short2((short)dx, (short)dy);
    }
}

// one 64-thread block per key line
__global__ void __launch_bounds__(64) lbd_describe_kernel(const short2* __restrict__ grad, int W, int H, int n_img,
                                                          const int32_t* __restrict__ kl_off, const float4* __restrict__ seg,
                                                          const float2* __restrict__ dir, const int32_t* __restrict__ npix,
                                                          uint8_t* __restrict__ out_desc) {
    __shared__ float s_rows[LBD_ROWS][8];   // per row: pgdL, ngdL, pgdL^2, ngdL^2, pgdO, ngdO, pgdO^2, ngdO^2 (scaled)
    __shared__ float s_band[LBD_BANDS][8];  // band sums, same order
    __shared__ float s_desc[LBD_DESC];
    __shared__ float s_scale[3];            // tempM, tempS, then the renormalisation factor
    const int line = blockIdx.x, t = threadIdx.x;
    int lo = 0, hi = n_img;                 // image of this line: kl_off[img] <= line < kl_off[img + 1]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (kl_off[mid] <= line) lo = mid; else hi = mid;
    }
    const short2* g = grad + (size_t)lo * W * H;
    const float4 sg = seg[line];
    const float2 dl = dir[line];            // (cosf, sinf) of the float direction
    const float dL0 = dl.x, dL1 = dl.y;
    const float dO0 = -dL1, dO1 = dL0;
    const int L = npix[line];
    const float hw = (float)((L - 1) / 2), hh = (float)LBD_HALF_H;
    const float midX = __fmul_rn(__fadd_rn(sg.x, sg.z), 0.5f), midY = __fmul_rn(__fadd_rn(sg.y, sg.w), 0.5f);
    if (t < LBD_ROWS) {
        const int h = t;
        float x0 = __fadd_rn(__fadd_rn(__fmul_rn(-dL0, hw), __fmul_rn(dL1, hh)), midX);
        float y0 = __fadd_rn(__fsub_rn(__fmul_rn(-dL1, hw), __fmul_rn(dL0, hh)), midY);
        for (int k = 0; k < h; ++k) {       // row starts accumulate: row h starts after h sequential updates
            x0 = __fsub_rn(x0, dL1);
            y0 = __fadd_rn(y0, dL0);
        }
        float pL = 0.f, nL = 0.f, pO = 0.f, nO = 0.f, sx = x0, sy = y0;
        for (int w = 0; w < L; ++w) {
            // (short) round(sCor), then clamped to the image
            int xc = (short)__float2int_rz(roundf(sx)), yc = (short)__float2int_rz(roundf(sy));
            xc = xc < 0 ? 0 : (xc > W - 1 ? W - 1 : xc);
            yc = yc < 0 ? 0 : (yc > H - 1 ? H - 1 : yc);
            const short2 d = g[(size_t)yc * W + xc];
            const float dx = (float)d.x, dy = (float)d.y;
            const float gDL = __fadd_rn(__fmul_rn(dx, dL0), __fmul_rn(dy, dL1));
            const float gDO = __fadd_rn(__fmul_rn(dx, dO0), __fmul_rn(dy, dO1));
            if (gDL > 0.f) pL = __fadd_rn(pL, gDL); else nL = __fsub_rn(nL, gDL);
            if (gDO > 0.f) pO = __fadd_rn(pO, gDO); else nO = __fsub_rn(nO, gDO);
            sx = __fadd_rn(sx, dL0);
            sy = __fadd_rn(sy, dL1);
        }
        const float c = c_coef_g[h];
        pL = __fmul_rn(c, pL); nL = __fmul_rn(c, nL); pO = __fmul_rn(c, pO); nO = __fmul_rn(c, nO);
        s_rows[h][0] = pL; s_rows[h][1] = nL; s_rows[h][2] = __fmul_rn(pL, pL); s_rows[h][3] = __fmul_rn(nL, nL);
        s_rows[h][4] = pO; s_rows[h][5] = nO; s_rows[h][6] = __fmul_rn(pO, pO); s_rows[h][7] = __fmul_rn(nO, nO);
    }
    __syncthreads();
    // band b takes band b-1's rows (weight gaussCoefL_[h % 7]), its own (+7) and band b+1's (+14), folded in ascending h
    for (int k = t; k < LBD_BANDS * 8; k += blockDim.x) {
        const int b = k >> 3, s = k & 7;
        const bool sq = (s & 2) != 0;
        float acc = 0.f;
        for (int nb = b - 1; nb <= b + 1; ++nb) {
            if (nb < 0 || nb >= LBD_BANDS) continue;
            const int woff = (nb - b + 1) * LBD_BAND_W;   // b-1: 0, b: 7, b+1: 14
            for (int r = 0; r < LBD_BAND_W; ++r) {
                const float c = c_coef_l[r + woff], x = s_rows[nb * LBD_BAND_W + r][s];
                acc = __fadd_rn(acc, sq ? __fmul_rn(__fmul_rn(c, c), x) : __fmul_rn(c, x));
            }
        }
        s_band[b][s] = acc;
    }
    __syncthreads();
    if (t < LBD_BANDS * 4) {                // mean and std of one (band, quantity): pgdL, ngdL, pgdO, ngdO
        const int b = t >> 2, q = t & 3;
        const int sum = (q >> 1) * 4 + (q & 1), sum2 = sum + 2;   // quantity q's sum and sum of squares in s_band
        const float invN = (b == 0 || b == LBD_BANDS - 1) ? (float)(1.0 / 14.0) : (float)(1.0 / 21.0);
        const float m = __fmul_rn(s_band[b][sum], invN);
        s_desc[8 * b + q] = m;
        s_desc[8 * b + q + 4] = __fsqrt_rn(__fsub_rn(__fmul_rn(s_band[b][sum2], invN), __fmul_rn(m, m)));
    }
    __syncthreads();
    if (t == 0) {                           // tempM over the means, tempS over the stds, in ascending index
        float m = 0.f, s = 0.f;
        for (int b = 0; b < LBD_BANDS; ++b) {
            for (int k = 0; k < 4; ++k) m = __fadd_rn(m, __fmul_rn(s_desc[8 * b + k], s_desc[8 * b + k]));
            for (int k = 4; k < 8; ++k) s = __fadd_rn(s, __fmul_rn(s_desc[8 * b + k], s_desc[8 * b + k]));
        }
        s_scale[0] = __fdiv_rn(1.f, __fsqrt_rn(m));
        s_scale[1] = __fdiv_rn(1.f, __fsqrt_rn(s));
    }
    __syncthreads();
    for (int k = t; k < LBD_DESC; k += blockDim.x) {
        float v = __fmul_rn(s_desc[k], s_scale[(k & 7) >> 2]);
        if ((double)v > 0.4) v = 0.4f;      // compared in double, as the reference does
        s_desc[k] = v;
    }
    __syncthreads();
    if (t == 0) {
        float s = 0.f;
        for (int k = 0; k < LBD_DESC; ++k) s = __fadd_rn(s, __fmul_rn(s_desc[k], s_desc[k]));
        s_scale[2] = __fdiv_rn(1.f, __fsqrt_rn(s));
    }
    __syncthreads();
    for (int k = t; k < LBD_DESC; k += blockDim.x) s_desc[k] = __fmul_rn(s_desc[k], s_scale[2]);
    __syncthreads();
    if (t < 32) {                           // byte t: bit i is band a's entry i > band b's entry i (NaN compares false)
        const float* fa = s_desc + 8 * c_comb[t][0];
        const float* fb = s_desc + 8 * c_comb[t][1];
        unsigned v = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) v |= (fa[i] > fb[i] ? 1u : 0u) << i;
        out_desc[(size_t)line * 32 + t] = (uint8_t)v;
    }
}

}  // namespace

cudaError_t lbd_upload_tables(const float* coef_g, const float* coef_l) {
    cudaError_t e = cudaMemcpyToSymbol(c_coef_g, coef_g, sizeof(float) * LBD_ROWS);
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_coef_l, coef_l, sizeof(float) * 3 * LBD_BAND_W);
    return e;
}

cudaError_t launch_lbd(int n_img, int W, int H, const uint8_t* images, const int32_t* kl_off, int n_lines, const float* seg,
                       const float2* dir, const int32_t* npix, short2* grad, uint8_t* out_desc, cudaStream_t s,
                       cudaEvent_t* ev, int* launches) {
    cudaEventRecord(ev[0], s);
    constexpr int max_z = 65535;            // gridDim.z limit: images go in slices of at most that many
    for (int i0 = 0; i0 < n_img; i0 += max_z) {
        const dim3 tiles((W + LBD_TILE_W - 1) / LBD_TILE_W, (H + LBD_TILE_H - 1) / LBD_TILE_H, min(max_z, n_img - i0));
        lbd_grad_kernel<<<tiles, 256, 0, s>>>(images, W, H, i0, kl_off, grad);
        ++*launches;
    }
    cudaEventRecord(ev[1], s);
    if (n_lines > 0) {
        lbd_describe_kernel<<<n_lines, 64, 0, s>>>(grad, W, H, n_img, kl_off, reinterpret_cast<const float4*>(seg), dir, npix,
                                                    out_desc);
        ++*launches;
    }
    cudaEventRecord(ev[2], s);
    return cudaGetLastError();
}

}  // namespace plstvo
