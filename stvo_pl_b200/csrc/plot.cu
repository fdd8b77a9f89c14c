// plot.cu — StereoFrame::plotStereoFrame (src/stereoFrame.cpp:618-663) for the new frames of a session call
// (plstvo_stereo_session_plot): the rectified left image in BGR, then cv::circle of every stereo point and cv::line of every
// stereo line in (B, G, R) = (0, 200, 0), byte for byte with OpenCV.
//   plot_base_kernel   one thread / 4 pixels of one frame   GRAY2BGR of the grey device copy, or the colour staging remapped
//                                                           channel by channel (remap.cuh) with alpha dropped
//   plot_draw_kernel   one thread / point or line of one frame   the clipped radius-3 circle, or the clipped 8-connected line
// Every draw writes the same three bytes, so threads that meet on a pixel write one value and the image does not depend on
// their order: no atomics and no ordering between the draws are needed.
#include "host.cuh"
#include "remap.cuh"

using namespace plstvo;

namespace {

// (dx, dy) of the pixels cv::circle sets for radius 3, thickness 1, LINE_8 (OpenCV's integer circle; outside the image a
// pixel is skipped, the others still drawn)
__constant__ int8_t CIRCLE_3[16][2] = {{-3, 0}, {-2, -2}, {-2, -1}, {-2, 1}, {-2, 2}, {-1, -2}, {-1, 2}, {0, -3},
                                       {0, 3},  {1, -2},  {1, 2},   {2, -2},  {2, -1}, {2, 1},   {2, 2},  {3, 0}};

// One thread writes 4 consecutive pixels (12 bytes) of frame blockIdx.y.  C == 1: src holds grey images, each value
// replicated (cvtColor GRAY2BGR).  C == 3 / 4: src holds C-channel images and frame z takes maps[z] (null: the first three
// channels as they are, else cv::remap of each); dropping alpha after the remap is cvtColor(BGRA2BGR).
template <int C>
__global__ void __launch_bounds__(256) plot_base_kernel(const uint8_t* __restrict__ src, const RemapMaps* __restrict__ maps,
                                                        int W, int H, uint8_t* __restrict__ dst) {
    const int z = (int)blockIdx.y;
    const size_t N = (size_t)W * H;
    const size_t p0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (p0 >= N) return;
    const int m = p0 + 4 <= N ? 4 : (int)(N - p0);
    const uint8_t* S = src + (size_t)z * N * C;
    RemapMaps mp{nullptr, nullptr};
    if constexpr (C > 1) mp = maps[z];
    uint32_t w[3] = {0, 0, 0};   // the 12 output bytes, little-endian
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (i >= m) break;
        const size_t p = p0 + i;
        uint32_t ch[3];
        if constexpr (C == 1) {
            ch[0] = ch[1] = ch[2] = __ldg(S + p);
        } else if (mp.m1) {
            remap_channels<C>(S, W, H, __ldg(mp.m1 + p), __ldg(mp.m2 + p), ch);
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) ch[c] = __ldg(S + p * C + c);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) w[(3 * i + c) >> 2] |= ch[c] << (8 * ((3 * i + c) & 3));
    }
    uint8_t* D = dst + ((size_t)z * N + p0) * 3;
    if (m == 4 && ((uintptr_t)D & 3) == 0) {
        uint32_t* D4 = reinterpret_cast<uint32_t*>(D);
        D4[0] = w[0]; D4[1] = w[1]; D4[2] = w[2];
    } else {
        for (int k = 0; k < 3 * m; ++k) D[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
    }
}

__device__ __forceinline__ void put_pixel(uint8_t* D, int W, int x, int y) {
    uint8_t* q = D + ((size_t)y * W + x) * 3;
    q[0] = 0; q[1] = 200; q[2] = 0;
}

// cv::clipLine(Size2l, Point2l&, Point2l&): the first end point is moved before the second, and the second's move reads the
// moved first one, so the result depends on the order of the ends.  (int64)(double) truncates, as the reference's cast does.
__device__ bool clip_line(long long W, long long H, long long& x1, long long& y1, long long& x2, long long& y2) {
    const long long right = W - 1, bottom = H - 1;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        long long a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += (long long)(__dmul_rn((double)(a - y1), (double)(x2 - x1)) / (double)(y2 - y1));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += (long long)(__dmul_rn((double)(a - y2), (double)(x2 - x1)) / (double)(y2 - y1));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += (long long)(__dmul_rn((double)(a - x1), (double)(y2 - y1)) / (double)(x2 - x1));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += (long long)(__dmul_rn((double)(a - x2), (double)(y2 - y1)) / (double)(x2 - x1));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

// cv::line(img, p1, p2, c, 1, LINE_8): cv::LineIterator(img, p1, p2, 8, leftToRight = true), clipped first where an end
// point lies outside, then Bresenham's walk with OpenCV's error terms from the left end point
__device__ void draw_line(uint8_t* D, int W, int H, int px1, int py1, int px2, int py2) {
    long long x1 = px1, y1 = py1, x2 = px2, y2 = py2;
    if ((unsigned)px1 >= (unsigned)W || (unsigned)py1 >= (unsigned)H || (unsigned)px2 >= (unsigned)W ||
        (unsigned)py2 >= (unsigned)H)
        if (!clip_line(W, H, x1, y1, x2, y2)) return;
    int ax = (int)x1, ay = (int)y1, bx = (int)x2, by = (int)y2;
    if (bx < ax) {
        int t = ax; ax = bx; bx = t;
        t = ay; ay = by; by = t;
    }
    int dx = bx - ax, dy = by - ay, sy = 1;
    if (dy < 0) {
        dy = -dy;
        sy = -1;
    }
    const bool vert = dy > dx;
    if (vert) {
        const int t = dx; dx = dy; dy = t;
    }
    int err = dx - 2 * dy;
    const int plus = 2 * dx, minus = -2 * dy;
    int x = ax, y = ay;
    for (int i = 0; i <= dx; ++i) {
        put_pixel(D, W, x, y);
        const bool minor = err < 0;
        err += minus + (minor ? plus : 0);
        if (vert) {
            y += sy;
            x += minor ? 1 : 0;
        } else {
            x += 1;
            y += minor ? sy : 0;
        }
    }
}

// Thread i of frame blockIdx.y draws the frame's point i (i < its points) or its line i - points: int() of the record's
// coordinates (toward zero) gives the Point the reference passes
__global__ void __launch_bounds__(128) plot_draw_kernel(const double2* __restrict__ pt_pl, const int32_t* __restrict__ pt_off,
                                                        const double2* __restrict__ spl, const double2* __restrict__ epl,
                                                        const int32_t* __restrict__ ls_off, int W, int H, uint8_t* __restrict__ dst) {
    const int z = (int)blockIdx.y;
    const int i = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    const int p0 = pt_off[z], np = pt_off[z + 1] - p0;
    const int l0 = ls_off[z], nl = ls_off[z + 1] - l0;
    uint8_t* D = dst + (size_t)z * W * H * 3;
    if (i < np) {
        const double2 c = pt_pl[p0 + i];
        const int cx = (int)c.x, cy = (int)c.y;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int x = cx + CIRCLE_3[k][0], y = cy + CIRCLE_3[k][1];
            if ((unsigned)x < (unsigned)W && (unsigned)y < (unsigned)H) put_pixel(D, W, x, y);
        }
    } else if (i - np < nl) {
        const double2 s = spl[l0 + i - np], e = epl[l0 + i - np];
        draw_line(D, W, H, (int)s.x, (int)s.y, (int)e.x, (int)e.y);
    }
}

}  // namespace

int plstvo::session_plot(PlContext* ctx, const SessionCall& c, int W, int H, const RecPtrs& rec,
                         const std::vector<int32_t>& pt_off, const std::vector<int32_t>& ls_off, const int32_t* d_pt_off,
                         const int32_t* d_ls_off, cudaStream_t s) {
    PlStereoSession* ss = c.ss;
    const int n = c.n;
    const size_t N = (size_t)W * H;
    const bool colour = c.plot_raw != nullptr;
    const int Ch = colour ? ss->rect->channels : 1;
    Arena a;
    const size_t o_img = a.take((size_t)n * N * 3), o_tab = a.take(colour ? (size_t)n * sizeof(RemapMaps) : 0);
    const size_t o_grey = a.take(c.plot_host ? (size_t)n * N : 0);
    CK(ctx, a.alloc(ss->plot_buf));
    const uint8_t* src = colour ? c.plot_raw : c.plot_grey;
    if (c.plot_host) {
        CK(ctx, a.up(o_grey, c.plot_host, (size_t)n * N, s));
        src = a.u8(o_grey);
    }
    if (colour) {   // each new frame's left maps: its stream's rectifier (cams sessions) or the session's
        std::vector<RemapMaps> tab((size_t)n, RemapMaps{nullptr, nullptr});
        for (int k = 0; k < n; ++k) {
            const PlRectifier* r = ss->rects.empty() ? ss->rect : ss->rects[(size_t)c.ids[k]];
            if (r->maps) tab[(size_t)k] = RemapMaps{r->m1[0], r->m2[0]};
        }
        CK(ctx, a.up(o_tab, tab.data(), tab.size() * sizeof(RemapMaps), s));
    }
    const dim3 grid_base((unsigned)((N + 4 * 256 - 1) / (4 * 256)), (unsigned)n);
    const RemapMaps* d_tab = a.at<const RemapMaps>(o_tab);
    uint8_t* img = a.u8(o_img);
    if (Ch == 1)
        plot_base_kernel<1><<<grid_base, 256, 0, s>>>(src, nullptr, W, H, img);
    else if (Ch == 3)
        plot_base_kernel<3><<<grid_base, 256, 0, s>>>(src, d_tab, W, H, img);
    else
        plot_base_kernel<4><<<grid_base, 256, 0, s>>>(src, d_tab, W, H, img);
    CK(ctx, cudaGetLastError());
    ++ctx->launches;
    int most = 0;   // draws of the busiest frame
    for (int k = 0; k < n; ++k) most = std::max(most, pt_off[(size_t)k + 1] - pt_off[(size_t)k] + ls_off[(size_t)k + 1] - ls_off[(size_t)k]);
    if (most == 0) return 0;
    plot_draw_kernel<<<dim3((unsigned)((most + 127) / 128), (unsigned)n), 128, 0, s>>>(
        rec.at<const double2>(PT_PL), d_pt_off, rec.at<const double2>(LS_SPL), rec.at<const double2>(LS_EPL), d_ls_off, W, H, img);
    CK(ctx, cudaGetLastError());
    ++ctx->launches;
    return 0;
}
