// lsd_oracle.cpp -- C++ restatement of OpenCV's LineSegmentDetector (the LSD_REFINE_NONE path), the reference's
// LSDDetectorC KeyLine step and detectLineFeatures' sort-and-truncate.  TEST INFRASTRUCTURE: the checker of
// stvo_pl_b200/csrc/lsd.cu, held stage by stage to cv2 by tests/test_ref_lsd.py.  C++ so that every std::sort is
// libstdc++'s introsort, as in cv2 and the reference.  Built with -ffp-contract=off.
//
// Stages, as cv2 4.13 computes them (scale != 1):
//  - blur: GaussianBlur(ksize 2h + 1, sigma), sigma = sigma_scale / scale if scale < 1 else sigma_scale,
//    h = ceil(sigma * sqrt(6 ln 10)).  A whole 8-bit image takes the fixed-point path: taps rounded to 8 fractional bits,
//    row pass then column pass in integers, (v + 2^15) >> 16; BORDER_REFLECT_101.
//  - resize(..., fx = fy = scale, INTER_LINEAR_EXACT): size cvRound(W * scale) x cvRound(H * scale), coordinate
//    (d + 0.5) / scale - 0.5 in double, 8-bit fixed-point bilinear, edge pixels replicated.
//  - gradient on the 2x2 block at (x, y), x < w - 1, y < h - 1: gx = DA + BC, gy = DA - BC, norm = sqrt((gx^2 + gy^2) / 4);
//    angle = fastAtan2(gx, -gy) (degrees, float) * pi / 180 if norm > quant / sin(ang_th), else NOTDEF.
//  - seeds: the (w - 1)(h - 1) pixels with bin int(norm * (n_bins - 1) / max_norm), in decreasing bin; see seed_order.
//  - region growing from each unused, defined seed; the region angle is fastAtan2 of the float sums of cos / sin;
//    regions smaller than -log_nt / log10(ang_th / 180) are dropped (their pixels stay used).
//  - rectangle: gradient-weighted centroid, inertia-matrix angle, extents along it; endpoints + 0.5, divided by scale.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

constexpr double kNotdef = -1024.0;
constexpr double kPi = 3.14159265358979323846;
constexpr double kDegToRad = kPi / 180.0;

int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

float fast_atan2(float y, float x) {
    const float s = (float)(180 / kPi);
    const float p1 = 0.9997878412794807f * s, p3 = -0.3258083974640975f * s, p5 = 0.1555786518463281f * s,
                p7 = -0.04432655554792128f * s;
    const float ax = std::fabs(x), ay = std::fabs(y), eps = (float)2.2204460492503131e-16;
    float a, c, c2;
    if (ax >= ay) {
        c = ay / (ax + eps);
        c2 = c * c;
        a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    } else {
        c = ax / (ay + eps);
        c2 = c * c;
        a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

struct Params {
    double scale, sigma_scale, quant, ang_th;
    int n_bins;
};

struct Region {
    int x, y;
    double modgrad;
};

struct Detector {
    Params P;
    int w = 0, h = 0;                  // the scaled image
    std::vector<uint8_t> img;          // the scaled image
    std::vector<double> angles, modgrad;
    std::vector<uint8_t> used;
    std::vector<int> seeds;            // pixel indices in seed order

    bool aligned(int x, int y, double theta, double prec) const {
        const double a = angles[(size_t)y * w + x];
        if (a == kNotdef) return false;
        double n = theta - a;
        if (n < 0) n = -n;
        if (n > (3 * kPi) / 2) {
            n -= 2 * kPi;
            if (n < 0) n = -n;
        }
        return n <= prec;
    }
};

}  // namespace

extern "C" {

// Blur half-width h and the 2h + 1 taps (8 fractional bits) of GaussianBlur's fixed-point kernel for `sigma`.
int orc_lsd_gauss_taps(double sigma, int* taps) {
    const int h = (int)std::ceil(sigma * std::sqrt(2 * 3 * std::log(10.0)));
    const int n = 2 * h + 1;
    std::vector<double> v(h);
    const double scale2 = -0.125 / (sigma * sigma);   // x runs over twice the tap offset: exp(-offset^2 / (2 sigma^2))
    double sum = 0;
    for (int i = 0, x = 1 - n; i < h; ++i, x += 2) {
        v[i] = std::exp((double)(x * x) * scale2);
        sum += v[i];
    }
    sum *= 2;
    sum += 1;
    const double mul = 1 / sum;
    // getGaussianKernelFixedPoint_ED: the side taps from the outside in, each rounding error carried into the next; the
    // centre takes what is left of 256
    double err = 0;
    int side = 0;
    for (int i = 0; i < h; ++i) {
        const double adj = v[i] * mul * 256.0 + err;
        const int t = (int)std::lrint(adj);
        err = adj - (double)t;
        taps[i] = taps[n - 1 - i] = t;
        side += t;
    }
    taps[h] = 256 - 2 * side;
    return h;
}

void orc_lsd_blur(const uint8_t* src, int w, int h, uint8_t* dst, int kh, const int* taps) {
    std::vector<uint32_t> rows((size_t)w * (h + 2 * kh));
    for (int y = -kh; y < h + kh; ++y) {
        const uint8_t* s = src + (size_t)reflect101(y, h) * w;
        uint32_t* r = rows.data() + (size_t)(y + kh) * w;
        for (int x = 0; x < w; ++x) {
            uint32_t acc = 0;
            for (int j = -kh; j <= kh; ++j) acc += (uint32_t)taps[j + kh] * s[reflect101(x + j, w)];
            r[x] = acc;
        }
    }
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            uint32_t acc = 0;
            for (int i = -kh; i <= kh; ++i) acc += (uint32_t)taps[i + kh] * rows[(size_t)(y + kh + i) * w + x];
            const uint32_t v = (acc + 0x8000u) >> 16;
            dst[(size_t)y * w + x] = (uint8_t)(v > 255 ? 255 : v);
        }
}

// cvRound(n * scale): the size resize() gives for fx = scale.
int orc_lsd_scaled_size(int n, double scale) { return (int)std::lrint((double)n * scale); }

static void linear_exact_coeffs(int src, int dst, double scale, int* ofs, int* c1) {
    const double inv = 1.0 / scale;
    for (int d = 0; d < dst; ++d) {
        const double f = inv * ((double)d + 0.5) - 0.5;
        const int i = (int)std::floor(f);
        if (i >= 0 && src > 1 && i < src - 1) {
            ofs[d] = i;
            c1[d] = (int)std::lrint((f - (double)i) * 256.0);
        } else {
            ofs[d] = (i >= 0 && src > 1) ? src - 1 : 0;
            c1[d] = 0;
        }
    }
}

void orc_lsd_resize(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh, double scale) {
    if (sw == dw && sh == dh) {
        std::memcpy(dst, src, (size_t)sw * sh);
        return;
    }
    std::vector<int> xo(dw), xc(dw), yo(dh), yc(dh);
    linear_exact_coeffs(sw, dw, scale, xo.data(), xc.data());
    linear_exact_coeffs(sh, dh, scale, yo.data(), yc.data());
    for (int y = 0; y < dh; ++y) {
        const uint8_t* r0 = src + (size_t)yo[y] * sw;
        const uint8_t* r1 = src + (size_t)(yo[y] + (yc[y] ? 1 : 0)) * sw;
        for (int x = 0; x < dw; ++x) {
            const int x0 = xo[x], x1 = x0 + (xc[x] ? 1 : 0);
            const uint32_t h0 = (uint32_t)(256 - xc[x]) * r0[x0] + (uint32_t)xc[x] * r0[x1];
            const uint32_t h1 = (uint32_t)(256 - xc[x]) * r1[x0] + (uint32_t)xc[x] * r1[x1];
            const uint32_t v = h0 * (uint32_t)(256 - yc[y]) + h1 * (uint32_t)yc[y];
            dst[(size_t)y * dw + x] = (uint8_t)((v + 0x8000u) >> 16);
        }
    }
}

// Raw LSD segments (x1, y1, x2, y2 in image coordinates) of one image, in detection order.  seed_order 0: std::sort
// on the bin alone (OpenCV's comparator); 1: decreasing bin, raster order within a bin.  Returns the segment count;
// writes at most `cap` segments.  Optional outputs: the scaled image (w_s * h_s bytes) and its size.
int orc_lsd_segments(const uint8_t* image, int W, int H, double scale, double sigma_scale, double quant, double ang_th,
                     int n_bins, int seed_order, int cap, float* seg, uint8_t* scaled_out, int* wh_out) {
    Detector D;
    D.P = {scale, sigma_scale, quant, ang_th, n_bins};
    if (scale != 1) {
        const double sigma = scale < 1 ? sigma_scale / scale : sigma_scale;
        const int kmax = (int)std::ceil(sigma * std::sqrt(2 * 3 * std::log(10.0)));
        std::vector<int> taps(2 * kmax + 1);
        const int kh = orc_lsd_gauss_taps(sigma, taps.data());
        std::vector<uint8_t> blurred((size_t)W * H);
        orc_lsd_blur(image, W, H, blurred.data(), kh, taps.data());
        D.w = orc_lsd_scaled_size(W, scale);
        D.h = orc_lsd_scaled_size(H, scale);
        D.img.resize((size_t)D.w * D.h);
        orc_lsd_resize(blurred.data(), W, H, D.img.data(), D.w, D.h, scale);
    } else {
        D.w = W;
        D.h = H;
        D.img.assign(image, image + (size_t)W * H);
    }
    const int w = D.w, h = D.h;
    if (scaled_out) std::memcpy(scaled_out, D.img.data(), D.img.size());
    if (wh_out) wh_out[0] = w, wh_out[1] = h;

    const double prec = kPi * ang_th / 180;
    const double p = ang_th / 180;
    const double rho = quant / std::sin(prec);
    const size_t N = (size_t)w * h;
    D.angles.assign(N, kNotdef);
    D.modgrad.assign(N, 0.0);
    double max_grad = -1;
    for (int y = 0; y < h - 1; ++y)
        for (int x = 0; x < w - 1; ++x) {
            const uint8_t* r0 = D.img.data() + (size_t)y * w;
            const uint8_t* r1 = r0 + w;
            const int DA = r1[x + 1] - r0[x], BC = r0[x + 1] - r1[x];
            const int gx = DA + BC, gy = DA - BC;
            const double norm = std::sqrt((gx * gx + gy * gy) / 4.0);
            D.modgrad[(size_t)y * w + x] = norm;
            if (norm > rho) {
                D.angles[(size_t)y * w + x] = fast_atan2((float)gx, (float)-gy) * kDegToRad;
                if (norm > max_grad) max_grad = norm;
            }
        }
    const double bin_coef = max_grad > 0 ? double(n_bins - 1) / max_grad : 0;
    struct NormPoint {
        int x, y, norm;
    };
    std::vector<NormPoint> pts;
    pts.reserve(N);
    for (int y = 0; y < h - 1; ++y)
        for (int x = 0; x < w - 1; ++x) pts.push_back({x, y, int(D.modgrad[(size_t)y * w + x] * bin_coef)});
    auto by_norm = [](const NormPoint& a, const NormPoint& b) { return a.norm > b.norm; };
    if (seed_order == 0) std::sort(pts.begin(), pts.end(), by_norm);
    else std::stable_sort(pts.begin(), pts.end(), by_norm);

    const double log_nt = 5 * (std::log10(double(w)) + std::log10(double(h))) / 2 + std::log10(11.0);
    const size_t min_reg_size = size_t(-log_nt / std::log10(p));
    D.used.assign(N, 0);
    std::vector<Region> reg;
    reg.reserve(N);
    int n_seg = 0;
    for (const NormPoint& s : pts) {
        const size_t si = (size_t)s.y * w + s.x;
        if (D.used[si] || D.angles[si] == kNotdef) continue;
        // region_grow
        reg.clear();
        double reg_angle = D.angles[si];
        reg.push_back({s.x, s.y, D.modgrad[si]});
        float sumdx = float(std::cos(reg_angle)), sumdy = float(std::sin(reg_angle));
        D.used[si] = 1;
        for (size_t i = 0; i < reg.size(); ++i) {
            const int rx = reg[i].x, ry = reg[i].y;
            const int x0 = std::max(rx - 1, 0), x1 = std::min(rx + 1, w - 1);
            const int y0 = std::max(ry - 1, 0), y1 = std::min(ry + 1, h - 1);
            for (int yy = y0; yy <= y1; ++yy)
                for (int xx = x0; xx <= x1; ++xx) {
                    const size_t q = (size_t)yy * w + xx;
                    if (D.used[q] || !D.aligned(xx, yy, reg_angle, prec)) continue;
                    D.used[q] = 1;
                    reg.push_back({xx, yy, D.modgrad[q]});
                    const float a = float(D.angles[q]);
                    sumdx += std::cos(a);
                    sumdy += std::sin(a);
                    reg_angle = fast_atan2(sumdy, sumdx) * kDegToRad;
                }
        }
        if (reg.size() < min_reg_size) continue;
        // region2rect
        double cx = 0, cy = 0, sum = 0;
        for (const Region& r : reg) {
            cx += double(r.x) * r.modgrad;
            cy += double(r.y) * r.modgrad;
            sum += r.modgrad;
        }
        cx /= sum;
        cy /= sum;
        double Ixx = 0, Iyy = 0, Ixy = 0;
        for (const Region& r : reg) {
            const double dx = double(r.x) - cx, dy = double(r.y) - cy;
            Ixx += dy * dy * r.modgrad;
            Iyy += dx * dx * r.modgrad;
            Ixy -= dx * dy * r.modgrad;
        }
        const double lambda = 0.5 * (Ixx + Iyy - std::sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
        double theta = std::fabs(Ixx) > std::fabs(Iyy) ? double(fast_atan2(float(lambda - Ixx), float(Ixy)))
                                                       : double(fast_atan2(float(Ixy), float(lambda - Iyy)));
        theta *= kDegToRad;
        double diff = theta - reg_angle;
        while (diff <= -kPi) diff += 2 * kPi;
        while (diff > kPi) diff -= 2 * kPi;
        if (std::fabs(diff) > prec) theta += kPi;
        const double dx = std::cos(theta), dy = std::sin(theta);
        double l_min = 0, l_max = 0;
        for (const Region& r : reg) {
            const double l = (double(r.x) - cx) * dx + (double(r.y) - cy) * dy;
            if (l > l_max) l_max = l;
            else if (l < l_min) l_min = l;
        }
        double x1 = cx + l_min * dx + 0.5, y1 = cy + l_min * dy + 0.5;
        double x2 = cx + l_max * dx + 0.5, y2 = cy + l_max * dy + 0.5;
        if (scale != 1) {
            x1 /= scale;
            y1 /= scale;
            x2 /= scale;
            y2 /= scale;
        }
        if (n_seg < cap) {
            float* o = seg + 4 * (size_t)n_seg;
            o[0] = float(x1), o[1] = float(y1), o[2] = float(x2), o[3] = float(y2);
        }
        ++n_seg;
    }
    return n_seg;
}

// cv::LineIterator(img, Point(start), Point(end)).count, 8-connected: the float endpoints are rounded half to even, and
// where a rounded endpoint leaves the image (an endpoint in [W - 0.5, W) rounds to W) the segment is first clipped to it
// with clipLine (Cohen-Sutherland on integers, the intersections truncated toward zero); 0 when nothing is left.
int orc_lsd_line_count(int W, int H, const float* e) {
    int64_t x1 = std::lrint(e[0]), y1 = std::lrint(e[1]), x2 = std::lrint(e[2]), y2 = std::lrint(e[3]);
    const int64_t right = W - 1, bottom = H - 1;
    if ((uint64_t)x1 >= (uint64_t)W || (uint64_t)x2 >= (uint64_t)W || (uint64_t)y1 >= (uint64_t)H ||
        (uint64_t)y2 >= (uint64_t)H) {
        int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
        int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            int64_t a;
            if (c1 & 12) {
                a = c1 < 8 ? 0 : bottom;
                x1 += (int64_t)((double)(a - y1) * (double)(x2 - x1) / (double)(y2 - y1));
                y1 = a;
                c1 = (x1 < 0) + (x1 > right) * 2;
            }
            if (c2 & 12) {
                a = c2 < 8 ? 0 : bottom;
                x2 += (int64_t)((double)(a - y2) * (double)(x2 - x1) / (double)(y2 - y1));
                y2 = a;
                c2 = (x2 < 0) + (x2 > right) * 2;
            }
            if ((c1 & c2) == 0 && (c1 | c2) != 0) {
                if (c1) {
                    a = c1 == 1 ? 0 : right;
                    y1 += (int64_t)((double)(a - x1) * (double)(y2 - y1) / (double)(x2 - x1));
                    x1 = a;
                    c1 = 0;
                }
                if (c2) {
                    a = c2 == 1 ? 0 : right;
                    y2 += (int64_t)((double)(a - x2) * (double)(y2 - y1) / (double)(x2 - x1));
                    x2 = a;
                    c2 = 0;
                }
            }
        }
        if (c1 | c2) return 0;
    }
    return (int)std::max(std::abs(x2 - x1), std::abs(y2 - y1)) + 1;
}

// The reference's KeyLine step over raw segments (LSDDetectorC::detectImpl, one octave) and detectLineFeatures'
// sort-and-truncate.  Writes the kept lines in output order: seg [4] (sPointInOctave / ePointInOctave), angle, npix,
// response, length.  Returns the count.
int orc_lsd_keylines_from_segments(int W, int H, int n_raw, const float* raw, double min_length, int n_features,
                                   float* seg, float* angle, int32_t* npix, float* response, float* length) {
    struct KL {
        float e[4], angle, response, length;
        int npix;
    };
    std::vector<KL> kls;
    for (int k = 0; k < n_raw; ++k) {
        float e[4] = {raw[4 * k], raw[4 * k + 1], raw[4 * k + 2], raw[4 * k + 3]};
        if (e[0] < 0) e[0] = 0;
        if (e[0] >= W) e[0] = (float)W - 1.0f;
        if (e[2] < 0) e[2] = 0;
        if (e[2] >= W) e[2] = (float)W - 1.0f;
        if (e[1] < 0) e[1] = 0;
        if (e[1] >= H) e[1] = (float)H - 1.0f;
        if (e[3] < 0) e[3] = 0;
        if (e[3] >= H) e[3] = (float)H - 1.0f;
        const double len = (float)std::sqrt(std::pow(e[0] - e[2], 2) + std::pow(e[1] - e[3], 2));
        if (!(len > min_length)) continue;
        KL kl;
        std::memcpy(kl.e, e, sizeof e);
        kl.length = (float)len;
        kl.npix = orc_lsd_line_count(W, H, e);
        kl.angle = atan2f(e[3] - e[1], e[2] - e[0]);
        kl.response = kl.length / (float)std::max(W, H);
        kls.push_back(kl);
    }
    if ((int)kls.size() > n_features && n_features != 0) {
        std::sort(kls.begin(), kls.end(), [](const KL& a, const KL& b) { return a.response > b.response; });
        kls.resize(n_features);
    }
    for (size_t k = 0; k < kls.size(); ++k) {
        std::memcpy(seg + 4 * k, kls[k].e, sizeof kls[k].e);
        angle[k] = kls[k].angle;
        npix[k] = kls[k].npix;
        response[k] = kls[k].response;
        length[k] = kls[k].length;
    }
    return (int)kls.size();
}

}  // extern "C"
