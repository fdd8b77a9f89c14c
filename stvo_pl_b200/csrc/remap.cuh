// remap.cuh — cv::remap's INTER_LINEAR on one pixel, shared by the rectifier's kernels (rectify.cu) and the session plot's
// base image (plot.cu), so both read the maps and round as OpenCV does in one place.
#pragma once

#include <cstdint>

namespace plstvo {

// cv::remap's fixed point (INTER_BITS 5, INTER_REMAP_COEF_BITS 15): the weights of the four taps are ((32 - ax)(32 - ay),
// ax (32 - ay), (32 - ax) ay, ax ay) * 32, OpenCV's INTER_LINEAR table exactly (each bilinear product is a multiple of
// 1/1024), and the result is (sum + 2^14) >> 15, which is (sum / 32 + 2^9) >> 10.  A tap outside the image reads 0.
__device__ __forceinline__ uint32_t remap_pixel(const uint8_t* __restrict__ S, int W, int H, short2 m, uint32_t f) {
    f &= 1023u;   // OpenCV indexes its table with map2 & (INTER_TAB_SIZE2 - 1)
    const int ax = (int)(f & 31u), ay = (int)(f >> 5);
    const int x = m.x, y = m.y;
    const bool x0 = (unsigned)x < (unsigned)W, x1 = (unsigned)(x + 1) < (unsigned)W;
    const bool y0 = (unsigned)y < (unsigned)H, y1 = (unsigned)(y + 1) < (unsigned)H;
    const uint8_t* r0 = S + (size_t)y * W + x;
    const int v00 = (x0 && y0) ? __ldg(r0) : 0, v01 = (x1 && y0) ? __ldg(r0 + 1) : 0;
    const int v10 = (x0 && y1) ? __ldg(r0 + W) : 0, v11 = (x1 && y1) ? __ldg(r0 + W + 1) : 0;
    const int sum = v00 * ((32 - ax) * (32 - ay)) + v01 * (ax * (32 - ay)) + v10 * ((32 - ax) * ay) + v11 * (ax * ay);
    return (uint32_t)((sum + 512) >> 10);
}

// remap_pixel on each of the first three channels of a C-channel image: cv::remap of a multi-channel image interpolates
// every channel with the same weights as the one-channel remap.  Alpha is not read: a 4-channel tap is one aligned 4-byte
// load, of which the top byte is dropped.
template <int C>
__device__ __forceinline__ void remap_channels(const uint8_t* __restrict__ S, int W, int H, short2 m, uint32_t f, uint32_t ch[3]) {
    f &= 1023u;
    const int ax = (int)(f & 31u), ay = (int)(f >> 5);
    const int x = m.x, y = m.y;
    const bool x0 = (unsigned)x < (unsigned)W, x1 = (unsigned)(x + 1) < (unsigned)W;
    const bool y0 = (unsigned)y < (unsigned)H, y1 = (unsigned)(y + 1) < (unsigned)H;
    const int w00 = (32 - ax) * (32 - ay), w01 = ax * (32 - ay), w10 = (32 - ax) * ay, w11 = ax * ay;
    const ptrdiff_t row = (ptrdiff_t)W * C;
    const uint8_t* r0 = S + ((ptrdiff_t)y * W + x) * C;
    if constexpr (C == 4) {
        const uint32_t t00 = (x0 && y0) ? __ldg(reinterpret_cast<const uint32_t*>(r0)) : 0u;
        const uint32_t t01 = (x1 && y0) ? __ldg(reinterpret_cast<const uint32_t*>(r0 + 4)) : 0u;
        const uint32_t t10 = (x0 && y1) ? __ldg(reinterpret_cast<const uint32_t*>(r0 + row)) : 0u;
        const uint32_t t11 = (x1 && y1) ? __ldg(reinterpret_cast<const uint32_t*>(r0 + row + 4)) : 0u;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int sh = 8 * c;
            const int sum = (int)((t00 >> sh) & 255u) * w00 + (int)((t01 >> sh) & 255u) * w01 +
                            (int)((t10 >> sh) & 255u) * w10 + (int)((t11 >> sh) & 255u) * w11;
            ch[c] = (uint32_t)((sum + 512) >> 10);
        }
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int v00 = (x0 && y0) ? __ldg(r0 + c) : 0, v01 = (x1 && y0) ? __ldg(r0 + C + c) : 0;
            const int v10 = (x0 && y1) ? __ldg(r0 + row + c) : 0, v11 = (x1 && y1) ? __ldg(r0 + row + C + c) : 0;
            ch[c] = (uint32_t)((v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11 + 512) >> 10);
        }
    }
}

}  // namespace plstvo
