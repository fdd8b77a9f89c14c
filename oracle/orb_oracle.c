/* orb_oracle.c -- C restatement of what OpenCV's ORB does once the key points are chosen (ORB::compute, and the
 * description half of ORB::detectAndCompute): the image pyramid, the border filter, the intensity-centroid angle and the
 * rotated-BRIEF descriptor.  TEST INFRASTRUCTURE: the checker of stvo_pl_b200/csrc/orb.cu, held stage by stage to cv2 by
 * tests/test_ref_orb.py.  Built with -ffp-contract=off: where OpenCV's own code fuses a multiply-add (the vector code of
 * the float blur, in its AVX2/FMA dispatch) the restatement spells fmaf.
 *
 * Stages, as cv2 4.13 computes them:
 *  - level sizes: cvRound(W * (1.f / s_l)), s_l = (float)pow(scale, l); level l is resized from level l - 1 with
 *    INTER_LINEAR_EXACT (8-bit fixed-point bilinear, edge pixels replicated).
 *  - border filter: a key point survives iff cvRound(x) in [edge, W - edge) and cvRound(y) in [edge, H - edge).
 *  - angle: intensity centroid over the radius-15 disc on the unblurred level at cvRound(pt * (1.f / s_l)), then fastAtan2.
 *  - blur: the level is a sub-matrix of OpenCV's pyramid buffer, so GaussianBlur(7x7, sigma 2) takes sepFilter2D's float
 *    path (the same as cv2.sepFilter2D with getGaussianKernel(7, 2, CV_32F) taps): the row pass fuses in its 32-pixel
 *    vector steps (x < w / 32 * 32) and not in its scalar tail, the column pass fuses throughout, then cvRound.  Pixels
 *    outside the level come from the buffer's BORDER_REFLECT_101 border of the unblurred level.
 *  - rBRIEF: 256 point pairs rotated by the angle (float cos / sin), cvRound'ed, compared on the blurred level (samples
 *    that leave the level read the unblurred border). */
#include <math.h>
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../stvo_pl_b200/csrc/orb_pattern.h"

static int round_even(float v) { return (int)lrintf(v); }   /* cvRound: half to even (default rounding mode) */

static int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

float orc_orb_level_scale(double scale_factor, int level) { return (float)pow(scale_factor, (double)level); }

void orc_orb_level_size(int W, int H, double scale_factor, int level, int* w, int* h) {
    const float inv = 1.f / orc_orb_level_scale(scale_factor, level);
    *w = round_even((float)W * inv);
    *h = round_even((float)H * inv);
}

/* INTER_LINEAR_EXACT coefficients of one axis: offset and the weight of the second tap, 8 fractional bits */
static void linear_exact_coeffs(int src, int dst, int* ofs, int* c1) {
    const double scale = 1.0 / ((double)dst / (double)src);
    for (int d = 0; d < dst; ++d) {
        const double f = scale * ((double)d + 0.5) - 0.5;
        const int i = (int)floor(f);
        if (i >= 0 && src > 1 && i < src - 1) {
            ofs[d] = i;
            c1[d] = (int)lrint((f - (double)i) * 256.0);
        } else {                                  /* left or right of the source: the edge pixel, weight one */
            ofs[d] = (i >= 0 && src > 1) ? src - 1 : 0;
            c1[d] = 0;
        }
    }
}

void orc_orb_resize(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh) {
    if (sw == dw && sh == dh) {
        memcpy(dst, src, (size_t)sw * sh);
        return;
    }
    int* xo = malloc(sizeof(int) * dw * 2);
    int* yo = malloc(sizeof(int) * dh * 2);
    int *xc = xo + dw, *yc = yo + dh;
    linear_exact_coeffs(sw, dw, xo, xc);
    linear_exact_coeffs(sh, dh, yo, yc);
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
    free(xo);
    free(yo);
}

/* getGaussianKernel(7, 2, CV_32F) */
static void gauss_taps(float k[7]) {
    double e[7], sum = 0;
    for (int i = 0; i < 7; ++i) {
        const double x = i - 3;
        e[i] = exp(-(x * x) / (2.0 * 2.0 * 2.0));
        sum += e[i];
    }
    const double s = 1.0 / sum;
    for (int i = 0; i < 7; ++i) k[i] = (float)(e[i] * s);
}

void orc_orb_blur(const uint8_t* src, int w, int h, uint8_t* dst) {
    float k[7];
    gauss_taps(k);
    float* rows = malloc(sizeof(float) * (size_t)w * (h + 6));
    for (int y = -3; y < h + 3; ++y) {
        const uint8_t* s = src + (size_t)reflect101(y, h) * w;
        float* r = rows + (size_t)(y + 3) * w;
        for (int x = 0; x < w; ++x) {   /* OpenCV's row filter: 32-pixel FMA vector steps, then an unfused scalar tail */
            float acc = 0.f;
            if (x < w / 32 * 32)
                for (int j = 0; j < 7; ++j) acc = fmaf(k[j], (float)s[reflect101(x + j - 3, w)], acc);
            else
                for (int j = 0; j < 7; ++j) acc = acc + k[j] * (float)s[reflect101(x + j - 3, w)];
            r[x] = acc;
        }
    }
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            const float* c = rows + (size_t)(y + 3) * w + x;
            float acc = k[3] * c[0];
            for (int i = 1; i <= 3; ++i) acc = fmaf(k[3 + i], c[(size_t)i * w] + c[-(ptrdiff_t)i * w], acc);
            const int v = round_even(acc);
            dst[(size_t)y * w + x] = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
        }
    free(rows);
}

float orc_fast_atan2(float y, float x) {
    const float s = (float)(180 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * s, p3 = -0.3258083974640975f * s, p5 = 0.1555786518463281f * s,
                p7 = -0.04432655554792128f * s;
    const float ax = fabsf(x), ay = fabsf(y), eps = (float)2.2204460492503131e-16;
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

/* end of each row of the radius-15 disc (ORB's umax) */
static void disc_umax(int umax[17]) {
    const int half = 15;
    const int vmax = (int)floor(half * sqrt(2.f) / 2 + 1), vmin = (int)ceil(half * sqrt(2.f) / 2);
    for (int v = 0; v <= vmax; ++v) umax[v] = (int)lrint(sqrt((double)half * half - v * v));
    for (int v = half, v0 = 0; v >= vmin; --v) {
        while (umax[v0] == umax[v0 + 1]) ++v0;
        umax[v] = v0;
        ++v0;
    }
}

static inline int px(const uint8_t* img, int w, int h, int x, int y) {
    return img[(size_t)reflect101(y, h) * w + reflect101(x, w)];
}

float orc_orb_ic_angle(const uint8_t* lvl, int w, int h, int cx, int cy) {
    int umax[17];
    disc_umax(umax);
    int m01 = 0, m10 = 0;
    for (int u = -15; u <= 15; ++u) m10 += u * px(lvl, w, h, cx + u, cy);
    for (int v = 1; v <= 15; ++v) {
        int vsum = 0;
        for (int u = -umax[v]; u <= umax[v]; ++u) {
            const int p = px(lvl, w, h, cx + u, cy + v), m = px(lvl, w, h, cx + u, cy - v);
            vsum += p - m;
            m10 += u * (p + m);
        }
        m01 += v * vsum;
    }
    return orc_fast_atan2((float)m01, (float)m10);
}

void orc_orb_describe(const uint8_t* raw, const uint8_t* blur, int w, int h, int cx, int cy, float angle_deg,
                      uint8_t* desc) {
    const float ang = angle_deg * (float)(3.14159265358979323846 / 180.f);
    const float a = (float)cos(ang), b = (float)sin(ang);
    for (int i = 0; i < 32; ++i) {
        int val = 0;
        for (int k = 0; k < 8; ++k) {
            const signed char* p = kOrbPattern31[8 * i + k];
            int v[2];
            for (int e = 0; e < 2; ++e) {
                const float fx = (float)p[2 * e], fy = (float)p[2 * e + 1];
                const float px_ = fx * a - fy * b, py_ = fx * b + fy * a;
                const int x = cx + round_even(px_), y = cy + round_even(py_);
                v[e] = (x >= 0 && x < w && y >= 0 && y < h) ? blur[(size_t)y * w + x] : px(raw, w, h, x, y);
            }
            val |= (v[0] < v[1]) << k;
        }
        desc[i] = (uint8_t)val;
    }
}

/* Level images of one picture, packed level after level: raw (unblurred) and blurred. Returns the number of bytes. */
size_t orc_orb_pyramid(const uint8_t* img, int W, int H, int n_levels, double scale_factor, uint8_t* raw, uint8_t* blur) {
    size_t off = 0, prev = 0;
    int pw = W, ph = H;
    for (int l = 0; l < n_levels; ++l) {
        int w, h;
        orc_orb_level_size(W, H, scale_factor, l, &w, &h);
        if (l == 0) memcpy(raw, img, (size_t)W * H);
        else orc_orb_resize(raw + prev, pw, ph, raw + off, w, h);
        if (blur && w > 0 && h > 0) orc_orb_blur(raw + off, w, h, blur + off);
        prev = off;
        off += (size_t)w * h;
        pw = w;
        ph = h;
    }
    return off;
}

size_t orc_orb_pyramid_bytes(int W, int H, int n_levels, double scale_factor) {
    size_t n = 0;
    for (int l = 0; l < n_levels; ++l) {
        int w, h;
        orc_orb_level_size(W, H, scale_factor, l, &w, &h);
        n += (size_t)w * h;
    }
    return n;
}

/* One image: survivors of the border filter in input order.  kp_angle == NULL: angles computed (detectAndCompute);
 * else taken as given (compute).  Returns the survivor count; out_* and src_idx hold the first `count` rows. */
int orc_orb_compute(int W, int H, int n_levels, double scale_factor, int edge, const uint8_t* img, int n_kp,
                    const float* kp_xy, const int32_t* kp_oct, const float* kp_angle, float* out_angle, uint8_t* out_desc,
                    int32_t* src_idx) {
    if (W <= 2 * edge || H <= 2 * edge) return 0;
    const size_t bytes = orc_orb_pyramid_bytes(W, H, n_levels, scale_factor);
    uint8_t* raw = malloc(bytes + 1);
    uint8_t* blur = malloc(bytes + 1);
    orc_orb_pyramid(img, W, H, n_levels, scale_factor, raw, blur);
    int n = 0;
    for (int i = 0; i < n_kp; ++i) {
        const float x = kp_xy[2 * i], y = kp_xy[2 * i + 1];
        const int rx = round_even(x), ry = round_even(y);
        if (!(rx >= edge && rx < W - edge && ry >= edge && ry < H - edge)) continue;
        const int l = kp_oct[i];
        size_t off = 0;
        int w = W, h = H;
        for (int q = 0; q <= l; ++q) {
            orc_orb_level_size(W, H, scale_factor, q, &w, &h);
            if (q < l) off += (size_t)w * h;
        }
        const float inv = 1.f / orc_orb_level_scale(scale_factor, l);
        const int cx = round_even(x * inv), cy = round_even(y * inv);
        const float ang = kp_angle ? kp_angle[i] : orc_orb_ic_angle(raw + off, w, h, cx, cy);
        if (out_angle) out_angle[n] = ang;
        if (out_desc) orc_orb_describe(raw + off, blur + off, w, h, cx, cy, ang, out_desc + (size_t)n * 32);
        if (src_idx) src_idx[n] = i;
        ++n;
    }
    free(raw);
    free(blur);
    return n;
}

/* n_img images of one size on `threads` host threads; image i's key points are rows kp_off[i] .. kp_off[i + 1] and its
 * survivors start at row kp_off[i] of every output (the device layout).  counts[i] = survivors of image i. */
typedef struct {
    int W, H, n_levels, edge, n_img, next;
    double scale;
    const uint8_t* images;
    const int32_t *kp_off, *kp_oct;
    const float *kp_xy, *kp_angle;
    float* out_angle;
    uint8_t* out_desc;
    int32_t *src_idx, *counts;
    pthread_mutex_t mu;
} OrbBatch;

static void* orb_worker(void* arg) {
    OrbBatch* b = arg;
    for (;;) {
        pthread_mutex_lock(&b->mu);
        const int i = b->next++;
        pthread_mutex_unlock(&b->mu);
        if (i >= b->n_img) return NULL;
        const int o = b->kp_off[i];
        b->counts[i] = orc_orb_compute(b->W, b->H, b->n_levels, b->scale, b->edge, b->images + (size_t)i * b->W * b->H,
                                       b->kp_off[i + 1] - o, b->kp_xy + 2 * (size_t)o, b->kp_oct + o,
                                       b->kp_angle ? b->kp_angle + o : NULL, b->out_angle + o, b->out_desc + 32 * (size_t)o,
                                       b->src_idx + o);
    }
}

void orc_orb_compute_batch(int W, int H, int n_levels, double scale_factor, int edge, int n_img, const uint8_t* images,
                           const int32_t* kp_off, const float* kp_xy, const int32_t* kp_oct, const float* kp_angle,
                           float* out_angle, uint8_t* out_desc, int32_t* src_idx, int32_t* counts, int threads) {
    OrbBatch b = {W, H, n_levels, edge, n_img, 0, scale_factor, images, kp_off, kp_oct, kp_xy, kp_angle, out_angle,
                  out_desc, src_idx, counts};
    pthread_mutex_init(&b.mu, NULL);
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t t[256];
    for (int k = 1; k < threads; ++k) pthread_create(&t[k], NULL, orb_worker, &b);
    orb_worker(&b);
    for (int k = 1; k < threads; ++k) pthread_join(t[k], NULL);
    pthread_mutex_destroy(&b.mu);
}
