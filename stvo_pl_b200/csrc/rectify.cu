// rectify.cu — PinholeStereoCamera::rectifyImagesLR (src/pinholeStereoCamera.cpp:196-208) on the device: the rig's
// undistort-rectify maps, built once on the host as OpenCV builds them and held in HBM, and cv::remap's INTER_LINEAR with
// BORDER_CONSTANT 0 on a batch of grey images.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>

#include "host.cuh"
#include "remap.cuh"

using namespace plstvo;

namespace {

// 4 bytes from 4-byte aligned D on, else byte by byte
__device__ __forceinline__ void store4(uint8_t* D, uint32_t v) {
    if (((uintptr_t)D & 3) == 0) {
        *reinterpret_cast<uint32_t*>(D) = v;
    } else {
        D[0] = (uint8_t)v; D[1] = (uint8_t)(v >> 8); D[2] = (uint8_t)(v >> 16); D[3] = (uint8_t)(v >> 24);
    }
}

// One thread writes 4 consecutive pixels of one image (flat index p0 .. p0 + 3 of W*H): one 16-byte map1 load, one 8-byte
// map2 load, 16 byte gathers on the read-only path and one 4-byte store where the output is 4-byte aligned.  blockIdx.y is
// the image within a slice of at most 65535 starting at z0.  TABLE: image z takes maps[2 (z % per_block) + side] instead of
// the launch's two map pairs, and an entry without maps copies the image.
template <bool TABLE>
__global__ void __launch_bounds__(256) rectify_remap_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                            const short2* __restrict__ m1l, const uint16_t* __restrict__ m2l,
                                                            const short2* __restrict__ m1r, const uint16_t* __restrict__ m2r,
                                                            int W, int H, int per_block, int z0, const RemapMaps* __restrict__ maps) {
    const int z = z0 + (int)blockIdx.y;
    const size_t N = (size_t)W * H;
    const size_t p0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (p0 >= N) return;
    const bool right = (z / per_block) & 1;
    const short2* m1 = right ? m1r : m1l;
    const uint16_t* m2 = right ? m2r : m2l;
    const uint8_t* S = src + (size_t)z * N;
    uint8_t* D = dst + (size_t)z * N + p0;
    if constexpr (TABLE) {
        const RemapMaps mp = maps[2 * (z % per_block) + (right ? 1 : 0)];
        m1 = mp.m1;
        m2 = mp.m2;
        if (!m1) {
            const size_t e = p0 + 4 <= N ? p0 + 4 : N;
            if (e - p0 == 4)
                store4(D, (uint32_t)S[p0] | (uint32_t)S[p0 + 1] << 8 | (uint32_t)S[p0 + 2] << 16 | (uint32_t)S[p0 + 3] << 24);
            else
                for (size_t p = p0; p < e; ++p) D[p - p0] = S[p];
            return;
        }
    }
    if (p0 + 4 <= N) {   // the maps start 256-byte aligned, so p0 % 4 == 0 aligns both vector loads
        const int4 a = __ldg(reinterpret_cast<const int4*>(m1 + p0));
        const uint2 b = __ldg(reinterpret_cast<const uint2*>(m2 + p0));
        short2 m[4];
        memcpy(m, &a, sizeof a);
        const uint32_t v = remap_pixel(S, W, H, m[0], b.x & 0xffffu) | remap_pixel(S, W, H, m[1], b.x >> 16) << 8 |
                           remap_pixel(S, W, H, m[2], b.y & 0xffffu) << 16 | remap_pixel(S, W, H, m[3], b.y >> 16) << 24;
        if (((uintptr_t)D & 3) == 0) {
            *reinterpret_cast<uint32_t*>(D) = v;
        } else {
            D[0] = (uint8_t)v; D[1] = (uint8_t)(v >> 8); D[2] = (uint8_t)(v >> 16); D[3] = (uint8_t)(v >> 24);
        }
    } else {
        for (size_t p = p0; p < N; ++p) D[p - p0] = (uint8_t)remap_pixel(S, W, H, __ldg(m1 + p), __ldg(m2 + p));
    }
}

// cv::cvtColor(COLOR_BGR2GRAY) on 8-bit data, as cv2 4.13 computes it for every BGR triple (with and without IPP): 15-bit
// coefficients that sum to 2^15, so B = G = R = v gives v back.
__device__ __forceinline__ uint32_t bgr_to_grey(uint32_t b, uint32_t g, uint32_t r) {
    return (3735u * b + 19235u * g + 9798u * r + (1u << 14)) >> 15;
}

// cv::cvtColor(COLOR_RGB2GRAY) on 8-bit data: the same fixed point with the first and third channels swapped.  The
// reference's FLD branch converts a colour image with it (src/stereoFrame.cpp:251) and LBD then reads that image.
__device__ __forceinline__ uint32_t rgb_to_grey(uint32_t r, uint32_t g, uint32_t b) { return bgr_to_grey(b, g, r); }

// Byte k of a run of little-endian words (k a compile-time constant once the callers' loops unroll).
__device__ __forceinline__ uint32_t byte_of(const uint32_t* w, int k) { return (w[k >> 2] >> (8 * (k & 3))) & 255u; }

// cvtColor alone on n pixels of C interleaved channels (B, G, R[, A]), the whole batch as one run: the conversion does not
// depend on where an image starts.  One thread converts 16 pixels: C 16-byte loads and one 16-byte store, all aligned
// because the staging and the output slots start 256-byte aligned; the last partial group goes pixel by pixel.
// RGB: the same pixels' rgb_to_grey also go to dst_rgb (read once, two bytes written per pixel).
template <int C, bool RGB = false>
__global__ void __launch_bounds__(256) color_convert_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t n,
                                                            uint8_t* __restrict__ dst_rgb) {
    const size_t p0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 16;
    if (p0 >= n) return;
    if (p0 + 16 <= n) {
        uint32_t w[4 * C];
#pragma unroll
        for (int k = 0; k < C; ++k) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + p0 * C) + k);
            w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
        }
        uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
        for (int i = 0; i < 16; ++i)
            o[i >> 2] |= bgr_to_grey(byte_of(w, C * i), byte_of(w, C * i + 1), byte_of(w, C * i + 2)) << (8 * (i & 3));
        *reinterpret_cast<uint4*>(dst + p0) = make_uint4(o[0], o[1], o[2], o[3]);
        if constexpr (RGB) {
            uint32_t q[4] = {0, 0, 0, 0};
#pragma unroll
            for (int i = 0; i < 16; ++i)
                q[i >> 2] |= rgb_to_grey(byte_of(w, C * i), byte_of(w, C * i + 1), byte_of(w, C * i + 2)) << (8 * (i & 3));
            *reinterpret_cast<uint4*>(dst_rgb + p0) = make_uint4(q[0], q[1], q[2], q[3]);
        }
    } else {
        for (size_t p = p0; p < n; ++p) {
            const uint8_t* s = src + p * C;
            dst[p] = (uint8_t)bgr_to_grey(__ldg(s), __ldg(s + 1), __ldg(s + 2));
            if constexpr (RGB) dst_rgb[p] = (uint8_t)rgb_to_grey(__ldg(s), __ldg(s + 1), __ldg(s + 2));
        }
    }
}

// remap_channels (remap.cuh), then the conversion: the reference converts the remapped image
template <int C>
__device__ __forceinline__ uint32_t remap_grey(const uint8_t* __restrict__ S, int W, int H, short2 m, uint32_t f) {
    uint32_t ch[3];
    remap_channels<C>(S, W, H, m, f, ch);
    return bgr_to_grey(ch[0], ch[1], ch[2]);
}

// rectify_remap_kernel's layout on C-channel images: one thread writes 4 consecutive grey pixels of one image from one
// 16-byte map1 load and one 8-byte map2 load; image z of the staging slot starts at z * W * H * C.
// TABLE: the maps of image z as in rectify_remap_kernel; an entry without maps converts the image only.
// RGB: each remapped (or unmapped) pixel's rgb_to_grey also goes to dst_rgb, at the same index as its dst byte.
template <int C, bool TABLE, bool RGB = false>
__global__ void __launch_bounds__(256) color_remap_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                          const short2* __restrict__ m1l, const uint16_t* __restrict__ m2l,
                                                          const short2* __restrict__ m1r, const uint16_t* __restrict__ m2r,
                                                          int W, int H, int per_block, int z0, const RemapMaps* __restrict__ maps,
                                                          uint8_t* __restrict__ dst_rgb) {
    const int z = z0 + (int)blockIdx.y;
    const size_t N = (size_t)W * H;
    const size_t p0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (p0 >= N) return;
    const bool right = (z / per_block) & 1;
    const short2* m1 = right ? m1r : m1l;
    const uint16_t* m2 = right ? m2r : m2l;
    const uint8_t* S = src + (size_t)z * N * C;
    uint8_t* D = dst + (size_t)z * N + p0;
    if constexpr (TABLE) {
        const RemapMaps mp = maps[2 * (z % per_block) + (right ? 1 : 0)];
        m1 = mp.m1;
        m2 = mp.m2;
        if (!m1) {
            const size_t e = p0 + 4 <= N ? p0 + 4 : N;
            uint32_t v = 0, v2 = 0;
            for (size_t p = p0; p < e; ++p) {
                const uint8_t* q = S + p * C;
                v |= bgr_to_grey(__ldg(q), __ldg(q + 1), __ldg(q + 2)) << (8 * (p - p0));
                if constexpr (RGB) v2 |= rgb_to_grey(__ldg(q), __ldg(q + 1), __ldg(q + 2)) << (8 * (p - p0));
            }
            if (e - p0 == 4) {
                store4(D, v);
                if constexpr (RGB) store4(dst_rgb + (size_t)z * N + p0, v2);
            } else {
                for (size_t p = p0; p < e; ++p) D[p - p0] = (uint8_t)(v >> (8 * (p - p0)));
                if constexpr (RGB)
                    for (size_t p = p0; p < e; ++p) dst_rgb[(size_t)z * N + p] = (uint8_t)(v2 >> (8 * (p - p0)));
            }
            return;
        }
    }
    if constexpr (RGB) {   // both conversions of each remapped pixel's three channels
        uint8_t* D2 = dst_rgb + (size_t)z * N + p0;
        if (p0 + 4 <= N) {   // the maps as the grey form loads them: one 16-byte map1 and one 8-byte map2 load
            const int4 a = __ldg(reinterpret_cast<const int4*>(m1 + p0));
            const uint2 b = __ldg(reinterpret_cast<const uint2*>(m2 + p0));
            short2 m[4];
            memcpy(m, &a, sizeof a);
            const uint32_t f[4] = {b.x & 0xffffu, b.x >> 16, b.y & 0xffffu, b.y >> 16};
            uint32_t v = 0, v2 = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                uint32_t ch[3];
                remap_channels<C>(S, W, H, m[i], f[i], ch);
                v |= bgr_to_grey(ch[0], ch[1], ch[2]) << (8 * i);
                v2 |= rgb_to_grey(ch[0], ch[1], ch[2]) << (8 * i);
            }
            store4(D, v);
            store4(D2, v2);
        } else {
            for (size_t p = p0; p < N; ++p) {
                uint32_t ch[3];
                remap_channels<C>(S, W, H, __ldg(m1 + p), __ldg(m2 + p), ch);
                D[p - p0] = (uint8_t)bgr_to_grey(ch[0], ch[1], ch[2]);
                D2[p - p0] = (uint8_t)rgb_to_grey(ch[0], ch[1], ch[2]);
            }
        }
        return;
    }
    if (p0 + 4 <= N) {
        const int4 a = __ldg(reinterpret_cast<const int4*>(m1 + p0));
        const uint2 b = __ldg(reinterpret_cast<const uint2*>(m2 + p0));
        short2 m[4];
        memcpy(m, &a, sizeof a);
        const uint32_t v = remap_grey<C>(S, W, H, m[0], b.x & 0xffffu) | remap_grey<C>(S, W, H, m[1], b.x >> 16) << 8 |
                           remap_grey<C>(S, W, H, m[2], b.y & 0xffffu) << 16 | remap_grey<C>(S, W, H, m[3], b.y >> 16) << 24;
        if (((uintptr_t)D & 3) == 0) {
            *reinterpret_cast<uint32_t*>(D) = v;
        } else {
            D[0] = (uint8_t)v; D[1] = (uint8_t)(v >> 8); D[2] = (uint8_t)(v >> 16); D[3] = (uint8_t)(v >> 24);
        }
    } else {
        for (size_t p = p0; p < N; ++p) D[p - p0] = (uint8_t)remap_grey<C>(S, W, H, __ldg(m1 + p), __ldg(m2 + p));
    }
}

// cvRound (saturate_cast<int>(double)) on x86-64: round half to even; cvtsd2si gives INT_MIN for a result outside int, and for NaN
int cv_round(double v) {
    const double r = nearbyint(v);
    return (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;
}

// The CV_16SC2 + CV_16UC1 words of one pixel.  OpenCV's vector loop (vec) packs iu >> 5 to short with saturation, its
// scalar loop truncates.
void store_map(double u, double v, bool vec, int16_t* m1, uint16_t* m2) {
    const int iu = cv_round(u * 32.0), iv = cv_round(v * 32.0);
    const int su = iu >> 5, sv = iv >> 5;
    m1[0] = vec ? (int16_t)std::min(std::max(su, -32768), 32767) : (int16_t)su;
    m1[1] = vec ? (int16_t)std::min(std::max(sv, -32768), 32767) : (int16_t)sv;
    *m2 = (uint16_t)((iv & 31) * 32 + (iu & 31));
}
}  // namespace

namespace plstvo {

cudaError_t launch_rectify_remap(int n_img, int per_block, int W, int H, const uint8_t* src, uint8_t* dst,
                                 const short2* const m1[2], const uint16_t* const m2[2], cudaStream_t s, int* launches,
                                 const RemapMaps* maps) {
    const size_t quads = ((size_t)W * H + 3) / 4;
    const unsigned gx = (unsigned)((quads + 255) / 256);
    for (int z0 = 0; z0 < n_img; z0 += 65535) {
        const int nz = std::min(n_img - z0, 65535);
        if (maps)
            rectify_remap_kernel<true><<<dim3(gx, (unsigned)nz), 256, 0, s>>>(src, dst, nullptr, nullptr, nullptr, nullptr, W, H,
                                                                              per_block, z0, maps);
        else
            rectify_remap_kernel<false><<<dim3(gx, (unsigned)nz), 256, 0, s>>>(src, dst, m1[0], m2[0], m1[1], m2[1], W, H,
                                                                               per_block, z0, nullptr);
        ++*launches;
    }
    return cudaGetLastError();
}

// The grey device copy of n_img colour images (C channels): color_convert_kernel without maps, color_remap_kernel with;
// with a map table (per-image maps or none) its instantiation that reads it.
// RGB: the instantiations that also write the COLOR_RGB2GRAY plane dst_rgb.
template <int C, bool RGB>
cudaError_t launch_color_prepare(int n_img, int per_block, int W, int H, bool maps, const uint8_t* src, uint8_t* dst,
                                 const short2* const m1[2], const uint16_t* const m2[2], cudaStream_t s, int* launches,
                                 const RemapMaps* table, uint8_t* dst_rgb) {
    if (table) {
        const size_t quads = ((size_t)W * H + 3) / 4;
        const unsigned gx = (unsigned)((quads + 255) / 256);
        for (int z0 = 0; z0 < n_img; z0 += 65535) {
            const int nz = std::min(n_img - z0, 65535);
            color_remap_kernel<C, true, RGB><<<dim3(gx, (unsigned)nz), 256, 0, s>>>(src, dst, nullptr, nullptr, nullptr, nullptr, W,
                                                                                     H, per_block, z0, table, dst_rgb);
            ++*launches;
        }
        return cudaGetLastError();
    }
    if (!maps) {
        const size_t groups = ((size_t)n_img * W * H + 15) / 16;
        color_convert_kernel<C, RGB><<<(unsigned)((groups + 255) / 256), 256, 0, s>>>(src, dst, (size_t)n_img * W * H, dst_rgb);
        ++*launches;
        return cudaGetLastError();
    }
    const size_t quads = ((size_t)W * H + 3) / 4;
    const unsigned gx = (unsigned)((quads + 255) / 256);
    for (int z0 = 0; z0 < n_img; z0 += 65535) {
        const int nz = std::min(n_img - z0, 65535);
        color_remap_kernel<C, false, RGB><<<dim3(gx, (unsigned)nz), 256, 0, s>>>(src, dst, m1[0], m2[0], m1[1], m2[1], W, H,
                                                                                  per_block, z0, nullptr, dst_rgb);
        ++*launches;
    }
    return cudaGetLastError();
}

int rectify_enqueue(PlContext* ctx, const PlRectifier* rect, int n_img, int per_block, const std::vector<ImgPart>& parts,
                    cudaStream_t s, const uint8_t** d_out, const PlRectifier* const* rects, const uint8_t** d_rgb,
                    const uint8_t** d_raw) {
    const int W = rect->width, H = rect->height, Ch = rect->channels;
    const size_t bytes = (size_t)n_img * W * H;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, ctx->rect_ev.create());
    std::vector<RemapMaps> table(rects ? 2 * (size_t)per_block : 0, RemapMaps{nullptr, nullptr});
    for (size_t k = 0; k < table.size() / 2; ++k)
        if (const PlRectifier* r = rects[k])
            if (r->maps)
                for (int side = 0; side < 2; ++side) table[2 * k + side] = RemapMaps{r->m1[side], r->m2[side]};
    Arena a;
    const bool rgb = d_rgb && Ch > 1;
    const size_t o_raw = a.take(bytes * Ch), o_out = a.take(bytes), o_tab = a.take(table.size() * sizeof(RemapMaps));
    const size_t o_rgb = a.take(rgb ? bytes : 0);
    CK(ctx, a.alloc(ctx->arena_rect));
    CK(ctx, a.up(o_tab, table.data(), table.size() * sizeof(RemapMaps), s));
    const RemapMaps* d_tab = rects ? a.at<RemapMaps>(o_tab) : nullptr;
    size_t o = o_raw;
    for (const ImgPart& ip : parts) {
        const size_t b = (size_t)ip.n * W * H * Ch;
        CK(ctx, a.up(o, ip.p, b, s));
        o += b;
    }
    int launches = 0;
    ctx->rect_ran = false;
    CK(ctx, cudaEventRecord(ctx->rect_ev[0], s));
    if (Ch == 1)
        CK(ctx, launch_rectify_remap(n_img, per_block, W, H, a.u8(o_raw), a.u8(o_out), rect->m1, rect->m2, s, &launches, d_tab));
    else if (Ch == 3 && rgb)
        CK(ctx, (launch_color_prepare<3, true>(n_img, per_block, W, H, rect->maps, a.u8(o_raw), a.u8(o_out), rect->m1, rect->m2,
                                              s, &launches, d_tab, a.u8(o_rgb))));
    else if (Ch == 3)
        CK(ctx, (launch_color_prepare<3, false>(n_img, per_block, W, H, rect->maps, a.u8(o_raw), a.u8(o_out), rect->m1, rect->m2,
                                               s, &launches, d_tab, nullptr)));
    else if (rgb)
        CK(ctx, (launch_color_prepare<4, true>(n_img, per_block, W, H, rect->maps, a.u8(o_raw), a.u8(o_out), rect->m1, rect->m2,
                                              s, &launches, d_tab, a.u8(o_rgb))));
    else
        CK(ctx, (launch_color_prepare<4, false>(n_img, per_block, W, H, rect->maps, a.u8(o_raw), a.u8(o_out), rect->m1, rect->m2,
                                               s, &launches, d_tab, nullptr)));
    CK(ctx, cudaEventRecord(ctx->rect_ev[1], s));
    ctx->rect_ran = true;
    ctx->launches += launches;
    *d_out = a.u8(o_out);
    if (d_rgb) *d_rgb = rgb ? a.u8(o_rgb) : nullptr;
    if (d_raw) *d_raw = a.u8(o_raw);
    return 0;
}

}  // namespace plstvo

extern "C" {

int plstvo_init_undistort_rectify_map(const PlRectifyModel* m, int width, int height, int16_t* map1, uint16_t* map2) {
    if (!m || !map1 || !map2) return PLSTVO_E_INVALID;
    if (width < 1 || width > 32767 || height < 1 || height > 32767) return PLSTVO_E_INVALID;
    const bool fisheye = m->model == 1;
    const int nd = (int)m->n_dist;
    if (!(m->model == 0 || fisheye) || (double)nd != m->n_dist) return PLSTVO_E_INVALID;
    if (fisheye ? nd != 4 : !(nd == 4 || nd == 5 || nd == 8)) return PLSTVO_E_INVALID;   // no thin prism or tilt
    // iR = (P[:, :3] R)^-1: the product summed left to right, the inverse in the cofactor form cv::invert(DECOMP_LU) takes for
    // 3x3 (the fisheye builder inverts by SVD, which gave the same maps on every rig it was compared on)
    const double* R = m->R;
    const double* P = m->P;
    double A[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[3 * i + j] = P[4 * i] * R[j] + P[4 * i + 1] * R[3 + j] + P[4 * i + 2] * R[6 + j];
    double d = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
    if (d == 0.0 || !std::isfinite(d)) return PLSTVO_E_INVALID;
    d = 1.0 / d;
    const double ir[9] = {(A[4] * A[8] - A[5] * A[7]) * d, (A[2] * A[7] - A[1] * A[8]) * d, (A[1] * A[5] - A[2] * A[4]) * d,
                          (A[5] * A[6] - A[3] * A[8]) * d, (A[0] * A[8] - A[2] * A[6]) * d, (A[2] * A[3] - A[0] * A[5]) * d,
                          (A[3] * A[7] - A[4] * A[6]) * d, (A[1] * A[6] - A[0] * A[7]) * d, (A[0] * A[4] - A[1] * A[3]) * d};
    const double fx = m->K[0], fy = m->K[4], u0 = m->K[2], v0 = m->K[5];   // the skew K[1] is not read, as in OpenCV
    double k[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int c = 0; c < nd; ++c) k[c] = m->D[c];
    if (!fisheye) {
        // cv::initUndistortRectifyMap: k1 k2 p1 p2 [k3 [k4 k5 k6]].  Its vector loop (AVX2: two 4-lane double vectors) takes
        // blocks of 8 pixels, lane j the block's start + j*ir[0]; the columns after the last block add ir[0] per pixel.
        const double k1 = k[0], k2 = k[1], p1 = k[2], p2 = k[3], k3 = k[4], k4 = k[5], k5 = k[6], k6 = k[7];
        const int vec_cols = width - width % 8;
        for (int i = 0; i < height; ++i) {
            int16_t* m1 = map1 + (size_t)i * width * 2;
            uint16_t* m2 = map2 + (size_t)i * width;
            double X = i * ir[1] + ir[2], Y = i * ir[4] + ir[5], Wc = i * ir[7] + ir[8];
            for (int j = 0; j < width;) {
                const bool vec = j < vec_cols;
                const int lanes = vec ? 8 : 1;
                for (int l = 0; l < lanes; ++l, ++j) {
                    const double _x = vec ? X + (double)l * ir[0] : X, _y = vec ? Y + (double)l * ir[3] : Y,
                                 _w = vec ? Wc + (double)l * ir[6] : Wc;
                    const double w = 1. / _w, x = _x * w, y = _y * w;
                    const double x2 = x * x, y2 = y * y;
                    const double r2 = x2 + y2, _2xy = 2 * x * y;
                    const double kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2);
                    const double xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2);
                    const double yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy;
                    store_map(fx * xd + u0, fy * yd + v0, vec, m1 + 2 * j, m2 + j);
                }
                X += (double)lanes * ir[0];
                Y += (double)lanes * ir[3];
                Wc += (double)lanes * ir[6];
            }
        }
    } else {
        // cv::fisheye::initUndistortRectifyMap: one scalar loop, the row's X, Y, W accumulated pixel by pixel
        for (int i = 0; i < height; ++i) {
            int16_t* m1 = map1 + (size_t)i * width * 2;
            uint16_t* m2 = map2 + (size_t)i * width;
            double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
            for (int j = 0; j < width; ++j) {
                double u, v;
                if (_w <= 0) {
                    u = (_x > 0) ? -INFINITY : INFINITY;
                    v = (_y > 0) ? -INFINITY : INFINITY;
                } else {
                    const double x = _x / _w, y = _y / _w;
                    const double r = sqrt(x * x + y * y);
                    const double theta = atan(r);
                    const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2,
                                 theta8 = theta4 * theta4;
                    const double theta_d = theta * (1 + k[0] * theta2 + k[1] * theta4 + k[2] * theta6 + k[3] * theta8);
                    const double scale = (r == 0) ? 1.0 : theta_d / r;
                    u = fx * x * scale + u0;
                    v = fy * y * scale + v0;
                }
                store_map(u, v, false, m1 + 2 * j, m2 + j);
                _x += ir[0];
                _y += ir[3];
                _w += ir[6];
            }
        }
    }
    return 0;
}

}  // extern "C"

namespace {
// A checked rectifier of `channels` with the four maps uploaded, or none (all four null), under the context's lock.
PlRectifier* rectifier_new(PlContext* ctx, int width, int height, int channels, const int16_t* map1_l, const uint16_t* map2_l,
                           const int16_t* map1_r, const uint16_t* map2_r) {
    if (cudaSetDevice(ctx->device) != cudaSuccess) {
        fail(ctx, PLSTVO_E_CUDA, "cudaSetDevice failed");
        return nullptr;
    }
    PlRectifier* r = new PlRectifier();
    r->ctx = ctx;
    r->width = width;
    r->height = height;
    r->channels = channels;
    r->maps = map1_l != nullptr;
    if (!r->maps) return r;
    const size_t N = (size_t)width * height;
    const bool shared = map1_l == map1_r && map2_l == map2_r;
    const int16_t* m1[2] = {map1_l, map1_r};
    const uint16_t* m2[2] = {map2_l, map2_r};
    for (int side = 0; side < (shared ? 1 : 2); ++side) {
        cudaError_t e = r->map1[side].ensure(N * 4);
        if (e == cudaSuccess) e = r->map2[side].ensure(N * 2);
        if (e == cudaSuccess) e = cudaMemcpy(r->map1[side].p, m1[side], N * 4, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(r->map2[side].p, m2[side], N * 2, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) {
            ctx->err = std::string("plstvo_rectifier_create: ") + cudaGetErrorString(e);
            delete r;
            return nullptr;
        }
        r->m1[side] = r->map1[side].as<const short2>();
        r->m2[side] = r->map2[side].as<const uint16_t>();
    }
    if (shared) {
        r->m1[1] = r->m1[0];
        r->m2[1] = r->m2[0];
    }
    return r;
}
}  // namespace

extern "C" {

PlRectifier* plstvo_rectifier_create(PlContext* ctx, int width, int height, const int16_t* map1_l, const uint16_t* map2_l,
                                     const int16_t* map1_r, const uint16_t* map2_r) {
    if (!ctx) return nullptr;
    LOCK(ctx);
    if (width < 1 || width > 32767 || height < 1 || height > 32767) {
        fail(ctx, PLSTVO_E_INVALID, "width and height must be 1..32767");
        return nullptr;
    }
    if (!map1_l || !map2_l || !map1_r || !map2_r) {
        fail(ctx, PLSTVO_E_INVALID, "null map");
        return nullptr;
    }
    return rectifier_new(ctx, width, height, 1, map1_l, map2_l, map1_r, map2_r);
}

PlRectifier* plstvo_rectifier_create_color(PlContext* ctx, int width, int height, int channels, const int16_t* map1_l,
                                           const uint16_t* map2_l, const int16_t* map1_r, const uint16_t* map2_r) {
    if (!ctx) return nullptr;
    LOCK(ctx);
    if (channels != 3 && channels != 4) {
        fail(ctx, PLSTVO_E_INVALID, "channels must be 3 (BGR) or 4 (BGRA)");
        return nullptr;
    }
    if (width < 1 || width > 32767 || height < 1 || height > 32767) {
        fail(ctx, PLSTVO_E_INVALID, "width and height must be 1..32767");
        return nullptr;
    }
    const int given = (map1_l != nullptr) + (map2_l != nullptr) + (map1_r != nullptr) + (map2_r != nullptr);
    if (given != 0 && given != 4) {
        fail(ctx, PLSTVO_E_INVALID, "maps must be all four or none");
        return nullptr;
    }
    return rectifier_new(ctx, width, height, channels, map1_l, map2_l, map1_r, map2_r);
}

void plstvo_rectifier_destroy(PlRectifier* rect) {
    if (!rect) return;
    {
        LOCK(rect->ctx);   // no call of the context is using the maps once the lock is held: every call that reads them blocks
        cudaSetDevice(rect->ctx->device);
        rect->map1[0].release(); rect->map1[1].release(); rect->map2[0].release(); rect->map2[1].release();
    }
    delete rect;
}

int plstvo_rectify_batch(PlContext* ctx, const PlRectifier* rect, int B, const uint8_t* img_l, const uint8_t* img_r,
                         uint8_t* out_l, uint8_t* out_r) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!rect || B < 0) return fail(ctx, PLSTVO_E_INVALID, "null rectifier or negative B");
    if (rect->ctx != ctx) return fail(ctx, PLSTVO_E_INVALID, "the rectifier belongs to another context");
    if (B == 0) return 0;
    if (!img_l || !img_r || !out_l || !out_r) return fail(ctx, PLSTVO_E_INVALID, "null image");
    cudaStream_t s = ctx->s_main;
    const uint8_t* d_out = nullptr;
    if (const int rc = rectify_enqueue(ctx, rect, 2 * B, B, {ImgPart{img_l, B}, ImgPart{img_r, B}}, s, &d_out)) return rc;
    const size_t bytes = (size_t)B * rect->width * rect->height;
    CK(ctx, cudaMemcpyAsync(out_l, d_out, bytes, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaMemcpyAsync(out_r, d_out + bytes, bytes, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

int plstvo_debug_color_planes(PlContext* ctx, const PlRectifier* rect, const PlRectifier* const* rects, int B,
                              const uint8_t* img_l, const uint8_t* img_r, uint8_t* grey, uint8_t* rgb) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!rect || !img_l || !img_r || !grey || !rgb) return fail(ctx, PLSTVO_E_INVALID, "null argument");
    if (B < 1) return fail(ctx, PLSTVO_E_INVALID, "B must be at least 1");
    if (rect->ctx != ctx) return fail(ctx, PLSTVO_E_INVALID, "the rectifier belongs to another context");
    if (rect->channels == 1) return fail(ctx, PLSTVO_E_INVALID, "a grey rectifier has no RGB plane");
    for (int b = 0; rects && b < B; ++b) {
        const PlRectifier* r = rects[b];
        if (!r) continue;
        if (r->ctx != ctx) return fail(ctx, PLSTVO_E_INVALID, "a table rectifier belongs to another context");
        if (r->width != rect->width || r->height != rect->height)
            return fail(ctx, PLSTVO_E_INVALID, "a table rectifier's size differs from rect's");
        if (r->channels != rect->channels) return fail(ctx, PLSTVO_E_INVALID, "a table rectifier's channels differ from rect's");
    }
    cudaStream_t s = ctx->s_main;
    const uint8_t *d_grey = nullptr, *d_rgb = nullptr;
    if (const int rc = rectify_enqueue(ctx, rect, 2 * B, B, {ImgPart{img_l, B}, ImgPart{img_r, B}}, s, &d_grey, rects, &d_rgb))
        return rc;
    const size_t bytes = 2 * (size_t)B * rect->width * rect->height;
    CK(ctx, cudaMemcpyAsync(grey, d_grey, bytes, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaMemcpyAsync(rgb, d_rgb, bytes, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

int plstvo_rectify_kernel_times(PlContext* ctx, float* ms1) {
    if (!ctx || !ms1) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!ctx->rect_ran) return fail(ctx, PLSTVO_E_INVALID, "no rectify call on this context yet");
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaEventElapsedTime(ms1, ctx->rect_ev[0], ctx->rect_ev[1]));
    return 0;
}

}  // extern "C"
