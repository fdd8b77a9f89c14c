// lsd.cu — LSD line segments (cv::LineSegmentDetector's LSD_REFINE_NONE path, cv2 4.13) on a batch of grey images of one
// size, bit-exact.  DESIGN.md §4 ("LSD") says why each stage is exact here and what holds each to cv2.  Every
// floating-point operation whose rounding reaches an output is spelled with an explicit rounding intrinsic, so nvcc forms
// no FMA the reference does not have.
//
//   blur + resize -> gradient (angle or NOTDEF, norm, per-image max) -> bins and a per-image histogram of the defined
//   pixels -> seed order (a stable counting sort, one warp per image: decreasing bin, raster order within a bin) ->
//   region growing, one sequential walk per image (every accepted pixel moves the region angle, so one region's growth is
//   sequential; the images run in parallel) with each kept region's centroid and angle -> [host: cos / sin of the angles] -> extents and
//   endpoints.
#include "common.cuh"

namespace plstvo {
namespace lsd {   // named (not anonymous): the kernels keep stable symbol names across builds

constexpr double kNotdef = -1024.0;
constexpr double kPi = 3.14159265358979323846;
constexpr double kDegToRad = kPi / 180.0;

__device__ __forceinline__ int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

// GaussianBlur's 8-bit fixed-point path: taps with 8 fractional bits, a row pass and a column pass in integers (exact in
// any order), then (v + 2^15) >> 16
__global__ void lsd_blur_kernel(const uint8_t* __restrict__ src, int W, int H, LsdTaps taps, uint8_t* __restrict__ dst) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, img = blockIdx.z;
    if (x >= W) return;
    const uint8_t* s = src + (size_t)img * W * H;
    uint32_t acc = 0;
    for (int i = -taps.kh; i <= taps.kh; ++i) {
        const uint8_t* row = s + (size_t)reflect101(y + i, H) * W;
        uint32_t r = 0;
        for (int j = -taps.kh; j <= taps.kh; ++j) r += (uint32_t)taps.t[j + taps.kh] * row[reflect101(x + j, W)];
        acc += (uint32_t)taps.t[i + taps.kh] * r;
    }
    dst[(size_t)img * W * H + (size_t)y * W + x] = (uint8_t)min((acc + 0x8000u) >> 16, 255u);
}

// INTER_LINEAR_EXACT tap of destination coordinate d: source offset and the second weight (8 fractional bits)
__device__ __forceinline__ void linear_exact(int d, int src, double inv, int& o, int& c) {
    const double f = __dsub_rn(__dmul_rn(inv, __dadd_rn((double)d, 0.5)), 0.5);
    const int i = (int)floor(f);
    if (i >= 0 && src > 1 && i < src - 1) {
        o = i;
        c = __double2int_rn(__dmul_rn(__dsub_rn(f, (double)i), 256.0));
    } else {
        o = (i >= 0 && src > 1) ? src - 1 : 0;
        c = 0;
    }
}

__global__ void lsd_resize_kernel(const uint8_t* __restrict__ src, int sw, int sh, int dw, int dh, double inv,
                                  uint8_t* __restrict__ dst) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, img = blockIdx.z;
    if (x >= dw) return;
    int xo, xc, yo, yc;
    linear_exact(x, sw, inv, xo, xc);
    linear_exact(y, sh, inv, yo, yc);
    const uint8_t* s = src + (size_t)img * sw * sh;
    const uint8_t* r0 = s + (size_t)yo * sw;
    const uint8_t* r1 = s + (size_t)(yo + (yc ? 1 : 0)) * sw;
    const int x1 = xo + (xc ? 1 : 0);
    const uint32_t h0 = (uint32_t)(256 - xc) * r0[xo] + (uint32_t)xc * r0[x1];
    const uint32_t h1 = (uint32_t)(256 - xc) * r1[xo] + (uint32_t)xc * r1[x1];
    const uint32_t v = h0 * (uint32_t)(256 - yc) + h1 * (uint32_t)yc;
    dst[(size_t)img * dw * dh + (size_t)y * dw + x] = (uint8_t)((v + 0x8000u) >> 16);
}

// Gradient of the 2x2 block at (x, y) (ll_angle): norm, and the angle with its trig-table code where norm > rho; the last
// row and column have no gradient.  max_bits[img]: the largest defined norm's bits (norms are >= 0, so their bits order
// like the values; 0 where no pixel is defined).
__global__ void lsd_grad_kernel(const uint8_t* __restrict__ scaled, int w, int h, double rho, double* __restrict__ angle,
                                double* __restrict__ modgrad, int32_t* __restrict__ code,
                                unsigned long long* __restrict__ max_bits) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, img = blockIdx.z;
    unsigned long long mine = 0;
    if (x < w) {
        const size_t N = (size_t)w * h, i = (size_t)img * N + (size_t)y * w + x;
        double a = kNotdef, norm = 0;
        int c = -1;
        if (x < w - 1 && y < h - 1) {
            const uint8_t* r0 = scaled + (size_t)img * N + (size_t)y * w;
            const uint8_t* r1 = r0 + w;
            const int DA = r1[x + 1] - r0[x], BC = r0[x + 1] - r1[x];
            const int gx = DA + BC, gy = DA - BC;
            norm = __dsqrt_rn(__ddiv_rn((double)(gx * gx + gy * gy), 4.0));
            if (norm > rho) {
                a = __dmul_rn((double)fast_atan2((float)gx, (float)-gy), kDegToRad);
                c = (gx + LSD_GRAD_MAX) * LSD_TRIG_SIDE + (gy + LSD_GRAD_MAX);
                mine = (unsigned long long)__double_as_longlong(norm);
            }
        }
        angle[i] = a;
        modgrad[i] = norm;
        code[i] = c;
    }
    for (int o = 16; o; o >>= 1) mine = max(mine, __shfl_xor_sync(0xffffffffu, mine, o));
    if ((threadIdx.x & 31) == 0 && mine) atomicMax(&max_bits[img], mine);
}

// Bin of every defined pixel, int(norm * (n_bins - 1) / max_norm), and the per-image histogram of the bins
__global__ void lsd_bin_kernel(int w, int h, int n_bins, const double* __restrict__ angle, const double* __restrict__ modgrad,
                               const unsigned long long* __restrict__ max_bits, int32_t* __restrict__ bin,
                               int32_t* __restrict__ hist) {
    extern __shared__ int32_t s_hist[];
    const int img = blockIdx.z;
    for (int b = threadIdx.x; b < n_bins; b += blockDim.x) s_hist[b] = 0;
    __syncthreads();
    const double mx = __longlong_as_double((long long)max_bits[img]);
    const double coef = mx > 0 ? __ddiv_rn((double)(n_bins - 1), mx) : 0.0;
    const size_t N = (size_t)w * h;
    const int y = blockIdx.y;
    for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < w; x += gridDim.x * blockDim.x) {
        const size_t i = (size_t)img * N + (size_t)y * w + x;
        if (angle[i] == kNotdef) continue;
        const int b = __double2int_rz(__dmul_rn(modgrad[i], coef));
        bin[i] = b;
        atomicAdd(&s_hist[b], 1);
    }
    __syncthreads();
    for (int b = threadIdx.x; b < n_bins; b += blockDim.x)
        if (s_hist[b]) atomicAdd(&hist[(size_t)img * n_bins + b], s_hist[b]);
}

// Seed order of one image (one warp): the defined pixels by decreasing bin, in raster order within a bin.  OpenCV's order
// is this one (DESIGN.md §4, "LSD seed order").  The warp walks the raster 32 pixels at a time; the lanes of one bin take
// consecutive slots in lane (raster) order from that bin's counter in shared memory, and its lowest lane advances it.
__global__ void __launch_bounds__(32) lsd_seed_kernel(int w, int h, int n_bins, const double* __restrict__ angle,
                                                      const int32_t* __restrict__ bin, const int32_t* __restrict__ hist,
                                                      int32_t* __restrict__ seeds, int32_t* __restrict__ n_seeds) {
    extern __shared__ int32_t s_next[];
    const int img = blockIdx.x, lane = threadIdx.x;
    const size_t N = (size_t)w * h;
    if (lane == 0) {
        int acc = 0;
        for (int b = n_bins - 1; b >= 0; --b) {
            s_next[b] = acc;
            acc += hist[(size_t)img * n_bins + b];
        }
        n_seeds[img] = acc;
    }
    __syncwarp();
    const double* a = angle + img * N;
    const int32_t* bn = bin + img * N;
    int32_t* out = seeds + img * N;
    const int wm = w - 1, total = (w > 1 && h > 1) ? (h - 1) * wm : 0;   // the pixels with a gradient
    for (int base = 0; base < total; base += 32) {
        const int k = base + lane;
        int b = -1, i = 0;
        if (k < total) {
            i = (k / wm) * w + k % wm;
            if (a[i] != kNotdef) b = bn[i];
        }
        const unsigned same = __match_any_sync(0xffffffffu, b);
        if (b >= 0) {
            const int first = s_next[b];
            __syncwarp(same);
            out[first + __popc(same & ((1u << lane) - 1u))] = i;
            if (lane == __ffs(same) - 1) s_next[b] = first + __popc(same);
        }
        __syncwarp();
    }
}

__device__ __forceinline__ bool aligned(double a, double theta, double prec) {   // isAligned for a defined angle
    double n = __dsub_rn(theta, a);
    if (n < 0) n = -n;
    if (n > (3 * kPi) / 2) {
        n = __dsub_rn(n, 2 * kPi);
        if (n < 0) n = -n;
    }
    return n <= prec;
}

// Region growing and the region's rectangle angle (region_grow, region2rect's centroid, get_theta), one thread per
// image, in seed order.  Kept regions (at least min_reg pixels) are written as LsdRegion records at img * reg_cap and
// their pixels at rpix[img * N + start ..]; a dropped region's pixels stay used.
__global__ void lsd_grow_kernel(int w, int h, double prec, int min_reg, int reg_cap, const double* __restrict__ angle,
                                const double* __restrict__ modgrad, const int32_t* __restrict__ code,
                                const float4* __restrict__ trig, const int32_t* __restrict__ seeds,
                                const int32_t* __restrict__ n_seeds, uint8_t* __restrict__ used, int32_t* __restrict__ rpix,
                                LsdRegion* __restrict__ regions, int32_t* __restrict__ n_regions) {
    const int img = blockIdx.x;
    const size_t N = (size_t)w * h;
    const double* A = angle + img * N;
    const double* G = modgrad + img * N;
    const int32_t* Cd = code + img * N;
    const int32_t* S = seeds + img * N;
    uint8_t* U = used + img * N;
    int32_t* R = rpix + img * N;
    LsdRegion* out = regions + (size_t)img * reg_cap;
    const int ns = n_seeds[img];
    int fill = 0, nreg = 0;
    for (int k = 0; k < ns; ++k) {
        const int s = S[k];
        if (U[s]) continue;
        const int start = fill;
        double reg_angle = A[s];
        const float4 t0 = trig[Cd[s]];
        float sumdx = t0.x, sumdy = t0.y;   // (float)cos / sin (double) of the seed's angle
        U[s] = 1;
        R[fill++] = s;
        for (int i = start; i < fill; ++i) {
            const int p = R[i], px = p % w, py = p / w;
            const int x0 = max(px - 1, 0), x1 = min(px + 1, w - 1), y0 = max(py - 1, 0), y1 = min(py + 1, h - 1);
            for (int yy = y0; yy <= y1; ++yy)
                for (int xx = x0; xx <= x1; ++xx) {
                    const int q = yy * w + xx;
                    if (U[q]) continue;
                    const double a = A[q];
                    if (a == kNotdef || !aligned(a, reg_angle, prec)) continue;
                    U[q] = 1;
                    R[fill++] = q;
                    const float4 t = trig[Cd[q]];   // cosf / sinf of the float angle
                    sumdx = __fadd_rn(sumdx, t.z);
                    sumdy = __fadd_rn(sumdy, t.w);
                    reg_angle = __dmul_rn((double)fast_atan2(sumdy, sumdx), kDegToRad);
                }
        }
        const int n = fill - start;
        if (n < min_reg) {
            fill = start;
            continue;
        }
        double cx = 0, cy = 0, sum = 0;
        for (int i = start; i < fill; ++i) {
            const int p = R[i];
            const double g = G[p];
            cx = __dadd_rn(cx, __dmul_rn((double)(p % w), g));
            cy = __dadd_rn(cy, __dmul_rn((double)(p / w), g));
            sum = __dadd_rn(sum, g);
        }
        cx = __ddiv_rn(cx, sum);
        cy = __ddiv_rn(cy, sum);
        double Ixx = 0, Iyy = 0, Ixy = 0;
        for (int i = start; i < fill; ++i) {
            const int p = R[i];
            const double g = G[p], dx = __dsub_rn((double)(p % w), cx), dy = __dsub_rn((double)(p / w), cy);
            Ixx = __dadd_rn(Ixx, __dmul_rn(__dmul_rn(dy, dy), g));
            Iyy = __dadd_rn(Iyy, __dmul_rn(__dmul_rn(dx, dx), g));
            Ixy = __dsub_rn(Ixy, __dmul_rn(__dmul_rn(dx, dy), g));
        }
        const double d = __dsub_rn(Ixx, Iyy);
        const double disc = __dadd_rn(__dmul_rn(d, d), __dmul_rn(__dmul_rn(4.0, Ixy), Ixy));
        const double lambda = __dmul_rn(0.5, __dsub_rn(__dadd_rn(Ixx, Iyy), __dsqrt_rn(disc)));
        const float th = fabs(Ixx) > fabs(Iyy) ? fast_atan2((float)__dsub_rn(lambda, Ixx), (float)Ixy)
                                               : fast_atan2((float)Ixy, (float)__dsub_rn(lambda, Iyy));
        double theta = __dmul_rn((double)th, kDegToRad);
        double diff = __dsub_rn(theta, reg_angle);
        while (diff <= -kPi) diff = __dadd_rn(diff, 2 * kPi);
        while (diff > kPi) diff = __dsub_rn(diff, 2 * kPi);
        if (fabs(diff) > prec) theta = __dadd_rn(theta, kPi);
        if (nreg < reg_cap) out[nreg] = LsdRegion{cx, cy, theta, start, n};
        ++nreg;
    }
    n_regions[img] = nreg;
}

// One warp per kept region (dense index r; image i's regions are r_off[i] .. r_off[i + 1]): extents along (dx, dy) =
// (cos, sin) of its angle, then the endpoints + 0.5, divided by scale, rounded to float.
__global__ void lsd_extent_kernel(int n_img, int w, int h, int reg_cap, double scale, const int32_t* __restrict__ r_off,
                                  const LsdRegion* __restrict__ regions, const double2* __restrict__ dir,
                                  const int32_t* __restrict__ rpix, float4* __restrict__ seg) {
    const int r = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (r >= r_off[n_img]) return;
    int lo = 0, hi = n_img;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (r_off[mid] <= r) lo = mid; else hi = mid;
    }
    const LsdRegion g = regions[(size_t)lo * reg_cap + (r - r_off[lo])];
    const double dx = dir[r].x, dy = dir[r].y;
    const int32_t* R = rpix + (size_t)lo * w * h + g.start;
    double l_min = 0, l_max = 0;
    for (int i = lane; i < g.count; i += 32) {
        const int p = R[i];
        const double l = __dadd_rn(__dmul_rn(__dsub_rn((double)(p % w), g.cx), dx),
                                   __dmul_rn(__dsub_rn((double)(p / w), g.cy), dy));
        l_max = fmax(l_max, l);
        l_min = fmin(l_min, l);
    }
    for (int o = 16; o; o >>= 1) {
        l_max = fmax(l_max, __shfl_xor_sync(0xffffffffu, l_max, o));
        l_min = fmin(l_min, __shfl_xor_sync(0xffffffffu, l_min, o));
    }
    if (lane) return;
    double x1 = __dadd_rn(__dadd_rn(g.cx, __dmul_rn(l_min, dx)), 0.5), y1 = __dadd_rn(__dadd_rn(g.cy, __dmul_rn(l_min, dy)), 0.5);
    double x2 = __dadd_rn(__dadd_rn(g.cx, __dmul_rn(l_max, dx)), 0.5), y2 = __dadd_rn(__dadd_rn(g.cy, __dmul_rn(l_max, dy)), 0.5);
    if (scale != 1) {
        x1 = __ddiv_rn(x1, scale);
        y1 = __ddiv_rn(y1, scale);
        x2 = __ddiv_rn(x2, scale);
        y2 = __ddiv_rn(y2, scale);
    }
    seg[r] = make_float4((float)x1, (float)y1, (float)x2, (float)y2);
}

}  // namespace lsd

using namespace lsd;

size_t lsd_scratch_bytes(int n_img, int w, int h) {   // per-pixel device arrays of launch_lsd_grow's scaled images
    return (size_t)n_img * w * h * (8 + 8 + 4 + 4 + 4 + 4 + 1);
}

cudaError_t launch_lsd_grow(const LsdLaunch& L, cudaStream_t s, cudaEvent_t* ev, int* launches) {
    const size_t N = (size_t)L.w * L.h, M = (size_t)L.n_img * N;
    // carve the scratch: angle, modgrad (double), code, bin, seeds, rpix (int32), used (uint8)
    uint8_t* p = L.scratch;
    double* angle = reinterpret_cast<double*>(p); p += M * 8;
    double* modgrad = reinterpret_cast<double*>(p); p += M * 8;
    int32_t* code = reinterpret_cast<int32_t*>(p); p += M * 4;
    int32_t* bin = reinterpret_cast<int32_t*>(p); p += M * 4;
    int32_t* seeds = reinterpret_cast<int32_t*>(p); p += M * 4;
    int32_t* rpix = reinterpret_cast<int32_t*>(p); p += M * 4;
    uint8_t* used = p;
    cudaError_t e;
    if ((e = cudaEventRecord(ev[0], s))) return e;
    const uint8_t* scaled = L.images;
    if (L.scale != 1) {
        const dim3 gb((L.W + 127) / 128, L.H, L.n_img), gr((L.w + 127) / 128, L.h, L.n_img);
        lsd_blur_kernel<<<gb, 128, 0, s>>>(L.images, L.W, L.H, L.taps, L.blurred);
        *launches += 1;
        scaled = L.blurred;
        if (L.w != L.W || L.h != L.H) {   // resize() copies when the size does not change
            lsd_resize_kernel<<<gr, 128, 0, s>>>(L.blurred, L.W, L.H, L.w, L.h, 1.0 / L.scale, L.scaled);
            *launches += 1;
            scaled = L.scaled;
        }
    }
    if ((e = cudaGetLastError())) return e;
    if ((e = cudaEventRecord(ev[1], s))) return e;
    if ((e = cudaMemsetAsync(L.max_bits, 0, (size_t)L.n_img * 8, s))) return e;
    if ((e = cudaMemsetAsync(L.hist, 0, (size_t)L.n_img * L.n_bins * 4, s))) return e;
    if ((e = cudaMemsetAsync(used, 0, M, s))) return e;
    const dim3 gg((L.w + 127) / 128, L.h, L.n_img);
    lsd_grad_kernel<<<gg, 128, 0, s>>>(scaled, L.w, L.h, L.rho, angle, modgrad, code, L.max_bits);
    lsd_bin_kernel<<<dim3(1, L.h, L.n_img), 256, (size_t)L.n_bins * 4, s>>>(L.w, L.h, L.n_bins, angle, modgrad, L.max_bits,
                                                                           bin, L.hist);
    lsd_seed_kernel<<<L.n_img, 32, (size_t)L.n_bins * 4, s>>>(L.w, L.h, L.n_bins, angle, bin, L.hist, seeds, L.n_seeds);
    *launches += 3;
    if ((e = cudaGetLastError())) return e;
    if ((e = cudaEventRecord(ev[2], s))) return e;
    lsd_grow_kernel<<<L.n_img, 1, 0, s>>>(L.w, L.h, L.prec, L.min_reg, L.reg_cap, angle, modgrad, code, L.trig, seeds,
                                          L.n_seeds, used, rpix, L.regions, L.n_regions);
    *launches += 1;
    if ((e = cudaGetLastError())) return e;
    return cudaEventRecord(ev[3], s);
}

cudaError_t launch_lsd_extent(const LsdLaunch& L, int n_reg, const int32_t* r_off, const double2* dir, float4* seg,
                              cudaStream_t s, int* launches) {
    const size_t M = (size_t)L.n_img * L.w * L.h;
    const int32_t* rpix = reinterpret_cast<const int32_t*>(L.scratch + M * (8 + 8 + 4 + 4 + 4));
    if (n_reg) {
        lsd_extent_kernel<<<(n_reg + 7) / 8, 256, 0, s>>>(L.n_img, L.w, L.h, L.reg_cap, L.scale, r_off, L.regions, dir, rpix, seg);
        *launches += 1;
    }
    return cudaGetLastError();
}

}  // namespace plstvo
