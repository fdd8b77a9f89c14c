// capi_features.cu — the C-ABI's feature extraction on the GPU: ORB description and detection (orb.cu), LBD description
// (lbd.cu), and pose tracking from stereo images, where both feed the stereo step and the tracker without leaving HBM.
#include <cfloat>
#include <climits>
#include <cstring>
#include <functional>

#include "host.cuh"

using namespace plstvo;

extern "C" {

/* ---- ORB description (orb.cu) ---- */
void plstvo_default_orb_config(PlOrbConfig* c) {
    if (!c) return;
    c->n_levels = 4; c->scale_factor = 1.2; c->edge_threshold = 19; c->patch_size = 31; c->wta_k = 2;
}

namespace {
// INTER_LINEAR_EXACT taps of one axis (cv::resize's bit-exact linear interpolation): [0, dst) source offsets, then
// [dst, 2 dst) the 8-bit weight of the second tap; 0 where the source position is left or right of the source (edge pixel)
void orb_linear_exact_table(int src, int dst, int32_t* t) {
    const double scale = 1.0 / ((double)dst / (double)src);
    for (int d = 0; d < dst; ++d) {
        const double f = scale * ((double)d + 0.5) - 0.5;
        const int i = (int)floor(f);
        if (i >= 0 && src > 1 && i < src - 1) {
            t[d] = i;
            t[dst + d] = (int32_t)lrint((f - (double)i) * 256.0);
        } else {
            t[d] = (i >= 0 && src > 1) ? src - 1 : 0;
            t[dst + d] = 0;
        }
    }
}

int orb_check_config(PlContext* ctx, const PlOrbConfig* cfg) {
    if (cfg->patch_size != 31) return fail(ctx, PLSTVO_E_INVALID, "patch_size must be 31");
    if (cfg->wta_k != 2) return fail(ctx, PLSTVO_E_INVALID, "wta_k must be 2");
    if (cfg->n_levels < 1 || cfg->n_levels > ORB_MAX_LEVELS) return fail(ctx, PLSTVO_E_INVALID, "n_levels must be 1..32");
    if (cfg->edge_threshold < 0) return fail(ctx, PLSTVO_E_INVALID, "negative edge_threshold");
    if (cfg->n_levels > 1 && !(cfg->scale_factor > 1.0 && cfg->scale_factor < 1e6))
        return fail(ctx, PLSTVO_E_INVALID, "scale_factor must be > 1");
    return 0;
}

// level sizes and offsets, blur taps and resize tables of the pyramid; false: a level of zero size
bool orb_levels(const PlOrbConfig* cfg, int width, int height, OrbDevLevels& L, std::vector<int32_t>& tabs,
                std::vector<size_t>& tab_off) {
    L = OrbDevLevels{};
    L.n = cfg->n_levels;
    for (int l = 0; l < L.n; ++l) {
        const float scale = (float)pow(cfg->scale_factor, (double)l);
        L.inv[l] = 1.f / scale;
        L.w[l] = (int)lrintf((float)width * L.inv[l]);
        L.h[l] = (int)lrintf((float)height * L.inv[l]);
        if (L.w[l] < 1 || L.h[l] < 1) return false;
        L.raw_off[l] = l ? L.raw_stride : 0;
        if (l) L.raw_stride += (size_t)L.w[l] * L.h[l];
        L.blur_off[l] = L.blur_stride;
        L.blur_stride += (size_t)L.w[l] * L.h[l];
    }
    {   // getGaussianKernel(7, 2, CV_32F)
        double e[7], sum = 0;
        for (int i = 0; i < 7; ++i) {
            e[i] = exp(-((double)(i - 3) * (i - 3)) / (2.0 * 2.0 * 2.0));
            sum += e[i];
        }
        for (int i = 0; i < 7; ++i) L.taps[i] = (float)(e[i] * (1.0 / sum));
    }
    tabs.clear();
    tab_off.assign(2 * (size_t)L.n, 0);
    for (int l = 1; l < L.n; ++l) {
        tab_off[2 * l] = tabs.size();
        tabs.resize(tabs.size() + 2 * (size_t)L.w[l]);
        orb_linear_exact_table(L.w[l - 1], L.w[l], tabs.data() + tab_off[2 * l]);
        tab_off[2 * l + 1] = tabs.size();
        tabs.resize(tabs.size() + 2 * (size_t)L.h[l]);
        orb_linear_exact_table(L.h[l - 1], L.h[l], tabs.data() + tab_off[2 * l + 1]);
    }
    return true;
}

// the launchers' rs_tab: device pointers of the x and y resize tables of levels 1 .. n - 1 (d_tabs: orb_levels' tabs uploaded)
std::vector<const int32_t*> orb_resize_tabs(const int32_t* d_tabs, const std::vector<size_t>& tab_off, int n) {
    std::vector<const int32_t*> rs_tab(2 * (size_t)n, nullptr);
    for (size_t k = 2; k < rs_tab.size(); ++k) rs_tab[k] = d_tabs + tab_off[k];
    return rs_tab;
}

cudaError_t orb_init(PlContext* ctx) {   // constant tables and timing events, once per context
    if (ctx->orb_tables) return cudaSuccess;
    cudaError_t e = orb_upload_tables();
    if (e == cudaSuccess) e = ctx->orb_ev.create();
    if (e == cudaSuccess) e = ctx->orb_det_ev.create();
    if (e == cudaSuccess) ctx->orb_tables = true;
    return e;
}
}  // namespace

int plstvo_orb_compute_batch(PlContext* ctx, const PlOrbConfig* cfg, int n_img, int width, int height, const uint8_t* images,
                             const int32_t* kp_off, const float* kp_xy, const int32_t* kp_octave, const float* kp_angle,
                             float* out_angle, uint8_t* out_desc, int32_t* src_idx, int32_t* counts) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!cfg || n_img < 0 || width < 0 || height < 0) return fail(ctx, PLSTVO_E_INVALID, "null config or negative size");
    if (const int rc = orb_check_config(ctx, cfg)) return rc;
    if (n_img == 0) return 0;
    const char* bad = "null images / offsets or kp_off[0] != 0";
    if (!images) return fail(ctx, PLSTVO_E_INVALID, bad);
    if (const int rc = check_offsets(ctx, n_img, {kp_off}, bad, "kp_off is not non-decreasing",
                                     "more than 65535 key points in one image"))
        return rc;
    const size_t N = (size_t)kp_off[n_img];
    if (N && (!kp_xy || !kp_octave || !out_angle || !out_desc || !src_idx))
        return fail(ctx, PLSTVO_E_INVALID, "null key point or output array");
    for (size_t k = 0; k < N; ++k)
        if (kp_octave[k] < 0 || kp_octave[k] >= cfg->n_levels) return fail(ctx, PLSTVO_E_INVALID, "octave outside [0, n_levels)");
    OrbDevLevels L{};
    std::vector<int32_t> tabs;
    std::vector<size_t> tab_off;
    if (!orb_levels(cfg, width, height, L, tabs, tab_off)) return fail(ctx, PLSTVO_E_INVALID, "a pyramid level has zero size");
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, orb_init(ctx));
    const size_t img_bytes = (size_t)n_img * width * height;
    Arena a;
    const size_t o_img = a.take(img_bytes), o_raw = a.take((size_t)n_img * L.raw_stride + 1);
    const size_t o_blur = a.take((size_t)n_img * L.blur_stride), o_tab = a.take(tabs.size() * 4 + 4);
    const size_t o_off = a.take((size_t)(n_img + 1) * 4), o_xy = a.take(N * 8), o_oct = a.take(N * 4), o_ang = a.take(N * 4);
    const size_t o_oang = a.take(N * 4), o_desc = a.take(N * 32), o_src = a.take(N * 4), o_cnt = a.take((size_t)n_img * 4);
    CK(ctx, a.alloc(ctx->arena_orb));
    cudaStream_t s = ctx->s_main;
    CK(ctx, a.up(o_img, images, img_bytes, s));
    CK(ctx, a.up(o_tab, tabs.data(), tabs.size() * 4, s));
    CK(ctx, a.up(o_off, kp_off, (size_t)(n_img + 1) * 4, s));
    CK(ctx, a.up(o_xy, kp_xy, N * 8, s));
    CK(ctx, a.up(o_oct, kp_octave, N * 4, s));
    CK(ctx, a.up(o_ang, kp_angle, N * 4, s));
    const std::vector<const int32_t*> rs_tab = orb_resize_tabs(a.i32(o_tab), tab_off, L.n);
    int launches = 0;
    CK(ctx, launch_orb(L, n_img, width, height, cfg->edge_threshold, a.u8(o_img), a.u8(o_raw), a.u8(o_blur), rs_tab.data(),
                       a.i32(o_off), (int)N, a.f32(o_xy), a.i32(o_oct), kp_angle ? a.f32(o_ang) : nullptr, a.i32(o_src),
                       a.i32(o_cnt), a.f32(o_oang), a.u8(o_desc), s, ctx->orb_ev.ev, &launches));
    ctx->orb_computed = true;
    ctx->launches += launches;
    std::vector<int32_t> cnt((size_t)n_img), src_dev(N);
    CK(ctx, a.down(cnt.data(), o_cnt, (size_t)n_img * 4, s));
    CK(ctx, a.down(src_dev.data(), o_src, N * 4, s));
    std::vector<float> ang_dev(N);
    std::vector<uint8_t> desc_dev(N * 32);
    CK(ctx, a.down(ang_dev.data(), o_oang, N * 4, s));
    CK(ctx, a.down(desc_dev.data(), o_desc, N * 32, s));
    CK(ctx, cudaStreamSynchronize(s));
    long total = 0;
    for (int i = 0; i < n_img; ++i) {   // survivors only: rows past counts[i] stay as the caller left them
        const size_t r0 = (size_t)kp_off[i], n = (size_t)cnt[i];
        if (n) {
            memcpy(out_angle + r0, ang_dev.data() + r0, n * 4);
            memcpy(out_desc + 32 * r0, desc_dev.data() + 32 * r0, n * 32);
            memcpy(src_idx + r0, src_dev.data() + r0, n * 4);
        }
        if (counts) counts[i] = cnt[i];
        total += cnt[i];
    }
    return (int)total;
}

int plstvo_orb_kernel_times(PlContext* ctx, float* ms3) {
    if (!ctx || !ms3) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!ctx->orb_computed) return fail(ctx, PLSTVO_E_INVALID, "no ORB call on this context yet");
    CK(ctx, cudaSetDevice(ctx->device));
    for (int k = 0; k < 3; ++k) CK(ctx, cudaEventElapsedTime(&ms3[k], ctx->orb_ev[k], ctx->orb_ev[k + 1]));
    return 0;
}

/* ---- LBD description (lbd.cu) ---- */
namespace {
cudaError_t lbd_init(PlContext* ctx) {   // coefficient tables and timing events, once per context
    if (ctx->lbd_tables) return cudaSuccess;
    // BinaryDescriptor's constructor (binary_descriptor_custom.cpp:217-259) with widthOfBand_ 7, NUM_OF_BANDS 9: the
    // centres and sigmas are integer divisions, the weights exp() in double, rounded to float where computeLBD reads them
    float coef_l[21], coef_g[63];
    double u = (7 * 3 - 1) / 2, sigma = (7 * 2 + 1) / 2, invsigma2 = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 21; ++i) {
        const double dis = i - u;
        coef_l[i] = (float)exp(dis * dis * invsigma2);
    }
    u = (9 * 7 - 1) / 2;
    sigma = u;
    invsigma2 = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 63; ++i) {
        const double dis = i - u;
        coef_g[i] = (float)exp(dis * dis * invsigma2);
    }
    cudaError_t e = lbd_upload_tables(coef_g, coef_l);
    if (e == cudaSuccess) e = ctx->lbd_ev.create();
    if (e == cudaSuccess) ctx->lbd_tables = true;
    return e;
}

// key lines of n_img consecutive images: kl_off [n_img + 1] and the per-line arrays
struct LineSrc {
    int n_img; const int32_t* off; const float* seg; const float* angle; const int32_t* npix;
};

// the key-line checks of plstvo_lbd_compute_batch on one LineSrc (the arrays only where lines exist)
int lbd_check_lines(PlContext* ctx, const LineSrc& l) {
    if (const int rc = check_offsets(ctx, l.n_img, {l.off}, "null offsets or kl_off[0] != 0", "kl_off is not non-decreasing",
                                     "more than 65535 key lines in one image"))
        return rc;
    const size_t N = (size_t)l.off[l.n_img];
    if (N && (!l.seg || !l.angle || !l.npix)) return fail(ctx, PLSTVO_E_INVALID, "null image or key line array");
    for (size_t k = 0; k < N; ++k)
        if (l.npix[k] < 1 || l.npix[k] > 32767) return fail(ctx, PLSTVO_E_INVALID, "numOfPixels must be 1..32767");
    return 0;
}

// Enqueues LBD description on stream s for checked key lines (parts, in image order; at least one line in all) of images of one
// size: either device images (d_img, ready once img_ready has completed) or host images that go into arena_lbd (img_parts).
// Leaves the key lines' segments (sPointInOctave, ePointInOctave as given) and descriptors in arena_lbd.
int lbd_enqueue(PlContext* ctx, int width, int height, const std::vector<LineSrc>& parts, const uint8_t* d_img,
                cudaEvent_t img_ready, const std::vector<ImgPart>& img_parts, cudaStream_t s, const float** d_seg,
                const uint8_t** d_desc) {
    int n_img = 0;
    std::vector<int32_t> off(1, 0);
    for (const LineSrc& l : parts) {
        for (int i = 0; i < l.n_img; ++i) off.push_back(off.back() + l.off[i + 1] - l.off[i]);
        n_img += l.n_img;
    }
    const size_t N = (size_t)off.back();
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, lbd_init(ctx));
    const size_t img_bytes = (size_t)n_img * width * height;
    Arena a;
    const size_t o_img = a.take(d_img ? 0 : img_bytes), o_grad = a.take(img_bytes * 4), o_off = a.take((size_t)(n_img + 1) * 4);
    const size_t o_seg = a.take(N * 16), o_dir = a.take(N * 8), o_npix = a.take(N * 4), o_desc = a.take(N * 32);
    CK(ctx, a.alloc(ctx->arena_lbd));
    if (!d_img) {
        size_t o = o_img;
        for (const ImgPart& ip : img_parts) {
            const size_t bytes = (size_t)ip.n * width * height;
            CK(ctx, cudaMemcpyAsync(a.u8(o), ip.p, bytes, cudaMemcpyHostToDevice, s));
            o += bytes;
        }
    }
    CK(ctx, cudaMemcpyAsync(a.u8(o_off), off.data(), (size_t)(n_img + 1) * 4, cudaMemcpyHostToDevice, s));
    // dL = (cos, sin) of the float angle.  The reference's unqualified cos(float) / sin(float) bind to std::cos(float) /
    // std::sin(float), the C library's cosf / sinf (its translation unit includes <math.h>, whose C++ form puts the float
    // overloads into the global namespace), and GCC merges the pair into sincosf.  They are evaluated here, with the same
    // library, because no device function rounds them the same way.
    std::vector<float> dir(2 * N);
    size_t r = 0;
    for (const LineSrc& l : parts) {
        const size_t n = (size_t)l.off[l.n_img];
        if (!n) continue;
        CK(ctx, cudaMemcpyAsync(a.u8(o_seg) + r * 16, l.seg, n * 16, cudaMemcpyHostToDevice, s));
        const float* kl_angle = l.angle;
        float* d = dir.data() + 2 * r;
        for (size_t k = 0; k < n; ++k) sincosf(kl_angle[k], &d[2 * k + 1], &d[2 * k]);
        r += n;
    }
    CK(ctx, cudaMemcpyAsync(a.u8(o_dir), dir.data(), N * 8, cudaMemcpyHostToDevice, s));
    r = 0;
    for (const LineSrc& l : parts) {
        const size_t n = (size_t)l.off[l.n_img];
        if (n) CK(ctx, cudaMemcpyAsync(a.u8(o_npix) + r * 4, l.npix, n * 4, cudaMemcpyHostToDevice, s));
        r += n;
    }
    if (d_img && img_ready) CK(ctx, cudaStreamWaitEvent(s, img_ready, 0));
    int launches = 0;
    CK(ctx, launch_lbd(n_img, width, height, d_img ? d_img : a.u8(o_img), a.i32(o_off), (int)N, a.f32(o_seg),
                       a.at<float2>(o_dir), a.i32(o_npix), a.at<short2>(o_grad), a.u8(o_desc), s, ctx->lbd_ev.ev, &launches));
    ctx->lbd_computed = true;
    ctx->launches += launches;
    *d_seg = a.f32(o_seg);
    *d_desc = a.u8(o_desc);
    return 0;
}
}  // namespace

int plstvo_lbd_compute_batch(PlContext* ctx, int n_img, int width, int height, const uint8_t* images, const int32_t* kl_off,
                             const float* kl_seg, const float* kl_angle, const int32_t* kl_npix, uint8_t* out_desc) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (n_img < 0) return fail(ctx, PLSTVO_E_INVALID, "negative n_img");
    // the reference indexes pixels and counts samples in short
    if (width < 1 || width > 32767 || height < 1 || height > 32767) return fail(ctx, PLSTVO_E_INVALID, "width and height must be 1..32767");
    if (n_img == 0) return 0;
    const LineSrc lines{n_img, kl_off, kl_seg, kl_angle, kl_npix};
    if (const int rc = lbd_check_lines(ctx, lines)) return rc;
    const size_t N = (size_t)kl_off[n_img];
    if (N == 0) return 0;
    if (!images || !out_desc) return fail(ctx, PLSTVO_E_INVALID, "null image or key line array");
    cudaStream_t s = ctx->s_main;
    const float* d_seg = nullptr;
    const uint8_t* d_desc = nullptr;
    if (const int rc = lbd_enqueue(ctx, width, height, {lines}, nullptr, nullptr, {ImgPart{images, n_img}}, s, &d_seg, &d_desc))
        return rc;
    CK(ctx, cudaMemcpyAsync(out_desc, d_desc, N * 32, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    return (int)N;
}

int plstvo_lbd_kernel_times(PlContext* ctx, float* ms2) {
    if (!ctx || !ms2) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!ctx->lbd_computed) return fail(ctx, PLSTVO_E_INVALID, "no LBD call on this context yet");
    CK(ctx, cudaSetDevice(ctx->device));
    for (int k = 0; k < 2; ++k) CK(ctx, cudaEventElapsedTime(&ms2[k], ctx->lbd_ev[k], ctx->lbd_ev[k + 1]));
    return 0;
}

/* ---- ORB key-point selection + description (orb.cu) ---- */
void plstvo_default_orb_detect_config(PlOrbDetectConfig* c) {
    if (!c) return;
    plstvo_default_orb_config(&c->orb);
    c->n_features = 1200; c->score_type = 1; c->fast_threshold = 20;
}

namespace {
int orb_detect_check(PlContext* ctx, const PlOrbDetectConfig* cfg) {
    if (const int rc = orb_check_config(ctx, &cfg->orb)) return rc;
    if (cfg->n_features < 0) return fail(ctx, PLSTVO_E_INVALID, "negative n_features");
    if (cfg->score_type != 0 && cfg->score_type != 1) return fail(ctx, PLSTVO_E_INVALID, "score_type must be 0 (Harris) or 1 (FAST)");
    return 0;
}

// ORB's pyramid for images of width x height under a checked detect config: oc (scale_factor rounded to float, as ORB::create
// takes it) and the levels' geometry and resize tables.  PLSTVO_E_INVALID where the pyramid cannot be built.
int orb_detect_levels(PlContext* ctx, const PlOrbDetectConfig* cfg, int width, int height, PlOrbConfig& oc, OrbDevLevels& L,
                      std::vector<int32_t>& tabs, std::vector<size_t>& tab_off) {
    oc = cfg->orb;
    oc.scale_factor = (double)(float)oc.scale_factor;   // ORB::create takes a float scale factor
    if (oc.n_levels > 1 && !(oc.scale_factor > 1.0)) return fail(ctx, PLSTVO_E_INVALID, "scale_factor must be > 1 in float");
    L = OrbDevLevels{};
    if (!orb_levels(&oc, width, height, L, tabs, tab_off)) return fail(ctx, PLSTVO_E_INVALID, "a pyramid level has zero size");
    return 0;
}

// key points of an ORB detect call, left in HBM (CSR by image, arena_orb_kp) with the host copy of the offsets
struct OrbDetected {
    std::vector<int32_t> off;   // [n_img + 1]; also written in full when the call fails with PLSTVO_E_TOO_LARGE
    const float *xy = nullptr, *angle = nullptr, *response = nullptr;
    const int32_t* octave = nullptr;
    const uint8_t* desc = nullptr;
};

// Enqueues detection and description of n_img (> 0) images on s_main, for a checked config and per-image FAST thresholds th
// (clamped here), or d_th: device thresholds in [0, 255] written on s_main, read as they are: either device images already
// written on s_main (d_img) or host images (parts, in order) that go up into arena_orb.  `beside` (optional) is called with the device images and an event that completes once they are on the device,
// after the pyramid and FAST launches are enqueued and before the first offsets readback blocks this thread: work enqueued
// there on another stream overlaps those stages.
int orb_detect_enqueue(PlContext* ctx, const PlOrbDetectConfig* cfg, int n_img, int width, int height, const uint8_t* d_img,
                       const std::vector<ImgPart>& parts, const int32_t* fast_th, int capacity,
                       const std::function<int(const uint8_t*, cudaEvent_t)>& beside, OrbDetected& out,
                       const int32_t* d_th = nullptr) {
    PlOrbConfig oc;
    OrbDevLevels L;
    std::vector<int32_t> tabs;
    std::vector<size_t> tab_off;
    if (const int rc = orb_detect_levels(ctx, cfg, width, height, oc, L, tabs, tab_off)) return rc;
    const int nl = L.n;
    const bool harris = cfg->score_type == 0;
    OrbDetectLevels D{};
    {   // the per-level budget, in float as ORB computes it
        const float factor = (float)(1.0 / oc.scale_factor);
        float nd = (float)cfg->n_features * (1.f - factor) / (1.f - (float)pow((double)factor, (double)nl));
        int sum = 0;
        for (int l = 0; l < nl; ++l) {
            int n = 0;
            if (l < nl - 1) {
                n = (int)lrintf(nd);
                sum += n;
                nd *= factor;
            } else {
                n = std::max(cfg->n_features - sum, 0);
            }
            D.keep1[l] = harris ? 2 * n : n;
            D.keep2[l] = n;
            D.row0[l + 1] = D.row0[l] + L.h[l];
            D.layer_scale[l] = (float)pow(oc.scale_factor, (double)l);
        }
        D.edge = cfg->orb.edge_threshold;
        const float hs = 1.f / (28 * 255.f);   // 1 / ((1 << 2) * blockSize * 255), blockSize 7
        D.harris_scale4 = hs * hs * hs * hs;
    }
    const int R = D.row0[nl];
    std::vector<int32_t> th(d_th ? 0 : (size_t)n_img);
    for (size_t i = 0; i < th.size(); ++i) th[i] = std::min(std::max(fast_th[i], 0), 255);
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, orb_init(ctx));
    const size_t img_bytes = (size_t)n_img * width * height, NL = (size_t)n_img * nl;
    Arena a;
    const size_t o_img = a.take(d_img ? 0 : img_bytes), o_raw = a.take((size_t)n_img * L.raw_stride + 1);
    const size_t o_blur = a.take((size_t)n_img * L.blur_stride), o_tab = a.take(tabs.size() * 4 + 4);
    const size_t o_score = a.take((size_t)n_img * L.blur_stride), o_hist = a.take(NL * 256 * 4), o_cut = a.take(NL * 4);
    const size_t o_rcnt = a.take((size_t)n_img * R * 4), o_rbase = a.take((size_t)n_img * (R + 1) * 4);
    const size_t o_icnt = a.take((size_t)n_img * 4), o_soff = a.take((size_t)(n_img + 1) * 4), o_th = a.take((size_t)n_img * 4);
    const size_t o_lkeep = a.take(NL * 4), o_ckey = a.take(NL * 4), o_hoff = a.take((size_t)(n_img + 1) * 4);
    const size_t o_hcnt = a.take((size_t)n_img * 4);
    CK(ctx, a.alloc(ctx->arena_orb));
    cudaStream_t s = ctx->s_main;
    const uint8_t* img = d_img ? d_img : a.u8(o_img);
    if (!d_img) {
        size_t o = o_img;
        for (const ImgPart& ip : parts) {
            const size_t bytes = (size_t)ip.n * width * height;
            CK(ctx, cudaMemcpyAsync(a.u8(o), ip.p, bytes, cudaMemcpyHostToDevice, s));
            o += bytes;
        }
    }
    cudaEvent_t uploaded = nullptr;
    if (beside) {
        uploaded = next_event(ctx);
        CK(ctx, cudaEventRecord(uploaded, s));
    }
    CK(ctx, a.up(o_tab, tabs.data(), tabs.size() * 4, s));
    CK(ctx, a.up(o_th, th.data(), th.size() * 4, s));
    const std::vector<const int32_t*> rs_tab = orb_resize_tabs(a.i32(o_tab), tab_off, nl);
    cudaEvent_t* ev = ctx->orb_det_ev.ev;   // [0] start, [1] pyramid + blur, [2] FAST + NMS, [3] selection, [4] angle + descriptor
    int launches = 0;
    CK(ctx, cudaEventRecord(ev[0], s));
    launch_orb_pyramid(L, n_img, img, a.u8(o_raw), a.u8(o_blur), rs_tab.data(), s, &launches);
    CK(ctx, cudaEventRecord(ev[1], s));
    launch_orb_fast_select(L, D, n_img, img, a.u8(o_raw), d_th ? d_th : a.i32(o_th), a.u8(o_score),
                           a.at<uint32_t>(o_hist), a.i32(o_cut), a.i32(o_rcnt), a.i32(o_rbase), a.i32(o_icnt), a.i32(o_soff), s,
                           ev[2], &launches);
    CK(ctx, cudaGetLastError());
    if (beside)
        if (const int rc = beside(img, uploaded)) return rc;
    std::vector<int32_t>& off = out.off;
    off.assign((size_t)n_img + 1, 0);
    CK(ctx, cudaMemcpyAsync(off.data(), a.i32(o_soff), off.size() * 4, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    ctx->launches += launches;
    launches = 0;
    ctx->orb_detected = true;
    // too many key points: the offsets in full (the caller sizes its buffers from them), no key points
    auto too_large = [&]() -> int {
        CK(ctx, cudaEventRecord(ev[3], s));
        CK(ctx, cudaEventRecord(ev[4], s));
        for (int i = 0; i < n_img; ++i)
            if (off[i + 1] - off[i] > PLSTVO_MAX_FEATURES) return fail(ctx, PLSTVO_E_TOO_LARGE, "more than 65535 key points in one image");
        if (off[n_img] > capacity) return fail(ctx, PLSTVO_E_TOO_LARGE, "more key points than capacity");
        return 0;
    };
    auto exceeds = [&]() {
        if (off[n_img] > capacity) return true;
        for (int i = 0; i < n_img; ++i)
            if (off[i + 1] - off[i] > PLSTVO_MAX_FEATURES) return true;
        return false;
    };
    if (!harris && exceeds()) return too_large();
    const size_t N1 = (size_t)off[n_img];
    Arena b;
    const size_t o_lxy = b.take(N1 * 8), o_xy = b.take(N1 * 8), o_oct = b.take(N1 * 4), o_resp = b.take(N1 * 4);
    const size_t o_rank = b.take(N1 * 4), o_hresp = b.take(harris ? N1 * 4 : 0), o_fxy = b.take(harris ? N1 * 8 : 0);
    const size_t o_foct = b.take(harris ? N1 * 4 : 0), o_fresp = b.take(harris ? N1 * 4 : 0);
    const size_t o_frank = b.take(harris ? N1 * 4 : 0), o_ang = b.take(N1 * 4), o_desc = b.take(N1 * 32);
    CK(ctx, b.alloc(ctx->arena_orb_kp));
    launch_orb_fast_write(L, D, n_img, a.u8(o_score), a.i32(o_cut), a.i32(o_rbase), a.i32(o_soff), b.at<int2>(o_lxy),
                          b.f32(o_xy), b.i32(o_oct), b.f32(o_resp), b.i32(o_rank), s, &launches);
    const int32_t *d_off = a.i32(o_soff), *d_cnt = a.i32(o_icnt), *d_oct = b.i32(o_oct), *d_rank = b.i32(o_rank);
    const float *d_xy = b.f32(o_xy), *d_resp = b.f32(o_resp);
    if (harris) {
        uint32_t* ckey = a.at<uint32_t>(o_ckey);
        launch_orb_harris_select(L, D, n_img, (int)N1, img, a.u8(o_raw), a.i32(o_rbase), a.i32(o_soff),
                                 b.at<int2>(o_lxy), b.i32(o_oct), b.f32(o_hresp), ckey, a.i32(o_lkeep), a.i32(o_hoff),
                                 a.i32(o_hcnt), s, &launches);
        CK(ctx, cudaGetLastError());
        CK(ctx, cudaMemcpyAsync(off.data(), a.i32(o_hoff), off.size() * 4, cudaMemcpyDeviceToHost, s));
        CK(ctx, cudaStreamSynchronize(s));
        ctx->launches += launches;
        launches = 0;
        if (exceeds()) return too_large();
        launch_orb_harris_write(L, D, n_img, a.i32(o_soff), b.f32(o_xy), b.i32(o_oct), b.f32(o_hresp), ckey, a.i32(o_hoff),
                                b.f32(o_fxy), b.i32(o_foct), b.f32(o_fresp), b.i32(o_frank), s, &launches);
        d_off = a.i32(o_hoff); d_cnt = a.i32(o_hcnt); d_oct = b.i32(o_foct); d_rank = b.i32(o_frank); d_xy = b.f32(o_fxy);
        d_resp = b.f32(o_fresp);
    }
    CK(ctx, cudaEventRecord(ev[3], s));
    const size_t N = (size_t)off[n_img];
    launch_orb_describe(L, n_img, img, a.u8(o_raw), a.u8(o_blur), d_off, (int)N, d_xy, d_oct, nullptr, d_rank, d_cnt,
                        b.f32(o_ang), b.u8(o_desc), s, &launches);
    CK(ctx, cudaEventRecord(ev[4], s));
    CK(ctx, cudaGetLastError());
    ctx->launches += launches;
    out.xy = d_xy; out.octave = d_oct; out.angle = b.f32(o_ang); out.response = d_resp; out.desc = b.u8(o_desc);
    return 0;
}
}  // namespace

int plstvo_orb_detect_and_compute_batch(PlContext* ctx, const PlOrbDetectConfig* cfg, int n_img, int width, int height,
                                        const uint8_t* images, const int32_t* fast_th, int capacity, int32_t* kp_off,
                                        float* kp_xy, int32_t* kp_octave, float* kp_angle, float* kp_response, uint8_t* desc) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!cfg || n_img < 0 || width < 0 || height < 0 || capacity < 0)
        return fail(ctx, PLSTVO_E_INVALID, "null config, negative size or negative capacity");
    if (const int rc = orb_detect_check(ctx, cfg)) return rc;
    if (!kp_off) return fail(ctx, PLSTVO_E_INVALID, "null kp_off");
    kp_off[0] = 0;
    if (n_img == 0) return 0;
    if (!images) return fail(ctx, PLSTVO_E_INVALID, "null images");
    std::vector<int32_t> th((size_t)n_img, cfg->fast_threshold);
    if (fast_th) std::copy(fast_th, fast_th + n_img, th.begin());
    OrbDetected o;
    const int rc = orb_detect_enqueue(ctx, cfg, n_img, width, height, nullptr, {ImgPart{images, n_img}}, th.data(), capacity, nullptr, o);
    if (rc == PLSTVO_E_TOO_LARGE && o.off.size() == (size_t)n_img + 1) memcpy(kp_off, o.off.data(), o.off.size() * 4);
    if (rc) return rc;
    const size_t N = (size_t)o.off[n_img];
    cudaStream_t s = ctx->s_main;
    auto down = [&](void* dst, const void* src, size_t bytes) -> cudaError_t {
        return (dst && bytes) ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s) : cudaSuccess;
    };
    CK(ctx, down(kp_xy, o.xy, N * 8));
    CK(ctx, down(kp_octave, o.octave, N * 4));
    CK(ctx, down(kp_angle, o.angle, N * 4));
    CK(ctx, down(kp_response, o.response, N * 4));
    CK(ctx, down(desc, o.desc, N * 32));
    CK(ctx, cudaStreamSynchronize(s));
    memcpy(kp_off, o.off.data(), o.off.size() * 4);
    return (int)N;
}


int plstvo_orb_detect_kernel_times(PlContext* ctx, float* ms4) {
    if (!ctx || !ms4) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!ctx->orb_detected) return fail(ctx, PLSTVO_E_INVALID, "no ORB detect call on this context yet");
    CK(ctx, cudaSetDevice(ctx->device));
    for (int k = 0; k < 4; ++k) CK(ctx, cudaEventElapsedTime(&ms4[k], ctx->orb_det_ev[k], ctx->orb_det_ev[k + 1]));
    return 0;
}

/* ---- LSD line detection (lsd.cu) ---- */
void plstvo_default_lsd_config(PlLsdConfig* c) {
    if (!c) return;
    c->refine = 0; c->scale = 1.2; c->sigma_scale = 0.6; c->quant = 2.0; c->ang_th = 22.5; c->n_bins = 1024;
    c->min_line_length = 0.025; c->n_features = 300;
}

namespace {
constexpr double kLsdPi = 3.14159265358979323846;

// cv::fastAtan2 on the host, for the trig table: x86-64's baseline has no FMA, so nothing here is fused (as in lsd.cu)
float host_fast_atan2(float y, float x) {
    const float deg = (float)(180 / kLsdPi);
    const float p1 = 0.9997878412794807f * deg, p3 = -0.3258083974640975f * deg, p5 = 0.1555786518463281f * deg,
                p7 = -0.04432655554792128f * deg;
    const float ax = fabsf(x), ay = fabsf(y), eps = (float)2.2204460492503131e-16;
    const bool wide = ax >= ay;
    const float c = wide ? ay / (ax + eps) : ax / (ay + eps), c2 = c * c;
    float a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    if (!wide) a = 90.f - a;
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

// Region growing moves the region angle by the float sums of cos / sin: the seed's (float)cos(double), and cosf / sinf of
// each accepted pixel's float angle.  No device function rounds these as the C library does, and a pixel's angle depends
// only on its gradient pair, so the four values of every pair are computed here once per context, with the same library.
cudaError_t lsd_init(PlContext* ctx) {
    if (ctx->lsd_trig.p) return cudaSuccess;
    std::vector<float4> t((size_t)LSD_TRIG_SIDE * LSD_TRIG_SIDE);
    for (int gx = -LSD_GRAD_MAX; gx <= LSD_GRAD_MAX; ++gx)
        for (int gy = -LSD_GRAD_MAX; gy <= LSD_GRAD_MAX; ++gy) {
            const double a = (double)host_fast_atan2((float)gx, (float)-gy) * (kLsdPi / 180.0);
            const float af = (float)a;
            t[(size_t)(gx + LSD_GRAD_MAX) * LSD_TRIG_SIDE + (gy + LSD_GRAD_MAX)] =
                make_float4((float)cos(a), (float)sin(a), cosf(af), sinf(af));
        }
    cudaError_t e = ctx->lsd_ev.create();
    if (e == cudaSuccess) e = ctx->lsd_trig.ensure(t.size() * sizeof(float4));
    if (e == cudaSuccess) e = cudaMemcpy(ctx->lsd_trig.p, t.data(), t.size() * sizeof(float4), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) ctx->lsd_trig.release();
    return e;
}

struct KeyLine {
    float seg[4], angle, response, length;
    int32_t npix;
};

// cv::LineIterator(img, Point(start), Point(end)).count, 8-connected.  The endpoints are rounded half to even; one in
// [W - 0.5, W) (or the same in y) rounds outside the image, and LineIterator then clips the segment with clipLine
// (Cohen-Sutherland on integers, intersections truncated toward zero) before counting; 0 when nothing is left.
int line_iterator_count(int W, int H, const float* e) {
    int64_t x1 = lrintf(e[0]), y1 = lrintf(e[1]), x2 = lrintf(e[2]), y2 = lrintf(e[3]);
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
    return (int)std::max(std::llabs(x2 - x1), std::llabs(y2 - y1)) + 1;
}

// The KeyLine both line branches build from a segment e (start x, y, end x, y) of a W x H image, octave 0: lineLength
// (float)sqrt(pow(dx, 2) + pow(dy, 2)) of the float differences (the squares are exact in double), angle atan2 of the float
// differences, response lineLength / max(cols, rows), numOfPixels LineIterator's count on e.  Unqualified atan2 of two
// floats binds to std::atan2(float, float) in both branches (LSDDetector_custom.cpp and stereoFrame.cpp include <math.h>'s
// C++ form and `using namespace std`), the C library's atan2f, evaluated here with the same library.
KeyLine key_line(int W, int H, const float* e) {
    KeyLine kl;
    memcpy(kl.seg, e, sizeof kl.seg);
    const double dx = (double)(e[0] - e[2]), dy = (double)(e[1] - e[3]);
    kl.length = (float)sqrt(dx * dx + dy * dy);
    kl.npix = line_iterator_count(W, H, e);
    kl.angle = atan2f(e[3] - e[1], e[2] - e[0]);
    kl.response = kl.length / (float)std::max(W, H);
    return kl;
}

// LSDDetectorC::detectImpl's KeyLine step for one octave (3rdparty/line_descriptor/src/LSDDetector_custom.cpp:266-308)
// and detectLineFeatures' sort-and-truncate (src/stereoFrame.cpp:232-241), on the host: a few hundred lines per image, and
// atan2f is the C library's.  std::sort is the reference's own (libstdc++) sort, so equal responses keep its order.
void lsd_keylines(int W, int H, const float4* raw, int n, double min_length, int n_features, std::vector<KeyLine>& out) {
    out.clear();
    for (int k = 0; k < n; ++k) {
        float e[4] = {raw[k].x, raw[k].y, raw[k].z, raw[k].w};
        for (int c = 0; c < 4; ++c) {   // checkLineExtremes
            const int lim = (c & 1) ? H : W;
            if (e[c] < 0) e[c] = 0;
            if (e[c] >= lim) e[c] = (float)lim - 1.0f;
        }
        const KeyLine kl = key_line(W, H, e);
        if (!((double)kl.length > min_length)) continue;
        out.push_back(kl);
    }
    if ((int)out.size() > n_features && n_features != 0) {
        std::sort(out.begin(), out.end(), [](const KeyLine& a, const KeyLine& b) { return a.response > b.response; });
        out.resize((size_t)n_features);
    }
}

// detectLineFeatures' FLD branch after fld->detect (src/stereoFrame.cpp:260-299): FastLineDetector's segments seg [n][4]
// sorted by sort_flines_by_length (include/auxiliar.h:149-154: sqrt(pow(d, 2.0) + ..) in double, strict >) where there are
// more than n_features (!= 0) of them, truncated, then each made a KeyLine on the unclamped endpoints.  The sort runs on the
// segments in the caller's order with libstdc++'s std::sort, as the reference sorts its vector<Vec4f>, so equal lengths
// land where the reference puts them.
void fld_keylines(int W, int H, const float* seg, int n, int n_features, std::vector<KeyLine>& out) {
    struct Seg {
        float v[4];
    };
    std::vector<Seg> s((size_t)n);
    if (n) memcpy(s.data(), seg, (size_t)n * sizeof(Seg));
    if (n > n_features && n_features != 0) {
        auto len = [](const Seg& a) { return sqrt(pow(a.v[0] - a.v[2], 2.0) + pow(a.v[1] - a.v[3], 2.0)); };
        std::sort(s.begin(), s.end(), [&](const Seg& a, const Seg& b) { return len(a) > len(b); });
        s.resize((size_t)n_features);
    }
    out.clear();
    for (const Seg& e : s) out.push_back(key_line(W, H, e.v));
}

int lsd_check_config(PlContext* ctx, const PlLsdConfig* c) {
    if (c->refine != 0) return fail(ctx, PLSTVO_E_INVALID, "lsd refine: only 0 (LSD_REFINE_NONE) is supported");
    if (!(c->scale > 0) || !std::isfinite(c->scale) || !(c->sigma_scale > 0) || !std::isfinite(c->sigma_scale) ||
        !(c->quant >= 0) || !std::isfinite(c->quant) || !(c->ang_th > 0 && c->ang_th < 180) || c->n_bins < 1 ||
        c->n_bins > 4096 || !(c->min_line_length >= 0) || !std::isfinite(c->min_line_length) || c->n_features < 0)
        return fail(ctx, PLSTVO_E_INVALID, "lsd parameter out of range");
    // resize() takes INTER_AREA instead of INTER_LINEAR_EXACT when 1 / scale is 2 (its "area fast" case), which differs at
    // the last row and column of odd sizes; that path is not built
    if (fabs(1.0 / c->scale - 2.0) < DBL_EPSILON) return fail(ctx, PLSTVO_E_INVALID, "lsd scale 0.5 is not supported");
    return 0;
}
// flsd's launch parameters for n_img images of width x height under a checked config: the blur taps and the scaled size
// (blur with sigma_scale, / scale when shrinking, half-width ceil(sigma * sqrt(2 * 3 * ln 10)), then resize), the gradient
// threshold, the smallest kept region and the region records per image.  PLSTVO_E_INVALID: a blur wider than 31 taps or a
// scaled size outside 1..32767.
int lsd_plan(PlContext* ctx, const PlLsdConfig* cfg, int n_img, int width, int height, LsdLaunch& L) {
    L = LsdLaunch{};
    L.n_img = n_img; L.W = width; L.H = height; L.scale = cfg->scale; L.n_bins = cfg->n_bins;
    L.w = width; L.h = height;
    if (cfg->scale != 1) {
        const double sigma = cfg->scale < 1 ? cfg->sigma_scale / cfg->scale : cfg->sigma_scale;
        const double kh = ceil(sigma * sqrt(2 * 3 * log(10.0)));
        if (!(kh <= LSD_MAX_KH)) return fail(ctx, PLSTVO_E_INVALID, "lsd blur wider than 31 taps");
        L.taps.kh = (int)kh;
        // getGaussianKernelBitExact: exp(-x^2 / (2 sigma^2)) normalised to sum 1, rounded to 8 fractional bits
        std::vector<double> v((size_t)L.taps.kh);
        const double scale2 = -0.125 / (sigma * sigma);
        double sum = 0;
        for (int i = 0, x = -2 * L.taps.kh; i < L.taps.kh; ++i, x += 2) sum += (v[(size_t)i] = exp((double)(x * x) * scale2));
        const double mul = 1 / (sum * 2 + 1);
        // getGaussianKernelFixedPoint_ED: the side taps from the outside in, each rounding error carried into the next; the
        // centre takes what is left of 256
        double err = 0;
        int side = 0;
        for (int i = 0; i < L.taps.kh; ++i) {
            const double adj = v[(size_t)i] * mul * 256.0 + err;
            const int t = (int)lrint(adj);
            err = adj - (double)t;
            L.taps.t[i] = L.taps.t[2 * L.taps.kh - i] = t;
            side += t;
        }
        L.taps.t[L.taps.kh] = 256 - 2 * side;
        const double ws = rint((double)width * cfg->scale), hs = rint((double)height * cfg->scale);
        if (!(ws >= 1 && ws <= 32767 && hs >= 1 && hs <= 32767)) return fail(ctx, PLSTVO_E_INVALID, "lsd scaled size must be 1..32767");
        L.w = (int)ws;
        L.h = (int)hs;
    }
    const double prec = kLsdPi * cfg->ang_th / 180, p = cfg->ang_th / 180;
    L.prec = prec;
    L.rho = cfg->quant / sin(prec);
    const double log_nt = 5 * (log10((double)L.w) + log10((double)L.h)) / 2 + log10(11.0);
    const double min_reg = -log_nt / log10(p);
    L.min_reg = min_reg >= (double)INT_MAX ? INT_MAX : (int)(size_t)min_reg;
    L.reg_cap = (int)((size_t)L.w * L.h / (size_t)std::max(L.min_reg, 1) + 1);
    return 0;
}

// Enqueues LSD's device half (blur and resize, gradient, seed order, region growing) on stream s for L.n_img (> 0) images of
// one size planned by lsd_plan: either device images (d_img, ready once img_ready has completed) or host images that go into
// arena_lsd (img_parts).  Sets L's device pointers; lsd_finish continues on the same stream.
int lsd_enqueue(PlContext* ctx, LsdLaunch& L, const uint8_t* d_img, cudaEvent_t img_ready, const std::vector<ImgPart>& img_parts,
                cudaStream_t s) {
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, lsd_init(ctx));
    const int n_img = L.n_img;
    const bool scaled = L.scale != 1;
    const size_t in_bytes = (size_t)n_img * L.W * L.H, N = (size_t)L.w * L.h;
    Arena a;
    const size_t o_img = a.take(d_img ? 0 : in_bytes), o_blur = a.take(scaled ? in_bytes : 0),
                 o_scaled = a.take(scaled ? (size_t)n_img * N : 0), o_scr = a.take(lsd_scratch_bytes(n_img, L.w, L.h)),
                 o_max = a.take((size_t)n_img * 8), o_hist = a.take((size_t)n_img * L.n_bins * 4), o_ns = a.take((size_t)n_img * 4),
                 o_reg = a.take((size_t)n_img * L.reg_cap * sizeof(LsdRegion)), o_nreg = a.take((size_t)n_img * 4);
    CK(ctx, a.alloc(ctx->arena_lsd));
    L.images = d_img ? d_img : a.u8(o_img); L.blurred = a.u8(o_blur); L.scaled = a.u8(o_scaled); L.scratch = a.u8(o_scr);
    L.max_bits = a.at<unsigned long long>(o_max); L.hist = a.i32(o_hist); L.n_seeds = a.i32(o_ns);
    L.trig = ctx->lsd_trig.as<const float4>(); L.regions = a.at<LsdRegion>(o_reg); L.n_regions = a.i32(o_nreg);
    if (!d_img) {
        size_t o = o_img;
        for (const ImgPart& ip : img_parts) {
            const size_t bytes = (size_t)ip.n * L.W * L.H;
            CK(ctx, a.up(o, ip.p, bytes, s));
            o += bytes;
        }
    } else if (img_ready) {
        CK(ctx, cudaStreamWaitEvent(s, img_ready, 0));
    }
    int launches = 0;
    ctx->lsd_ran = false;   // until lsd_finish has recorded the rest of this call's events
    CK(ctx, launch_lsd_grow(L, s, ctx->lsd_ev.ev, &launches));
    ctx->launches += launches;
    return 0;
}

// The host continuation of lsd_enqueue, on the same stream: the region counts and records come down, the C library's cos /
// sin of the region angles go up (region2rect's dx, dy, as in the reference), the rectangles' raw segments come down, then
// the KeyLine step and the truncation run per image.  kls[i]: image i's key lines in the reference's order.  Returns with s
// synchronised.
int lsd_finish(PlContext* ctx, const PlLsdConfig* cfg, const LsdLaunch& L, cudaStream_t s, std::vector<std::vector<KeyLine>>& kls) {
    const int n_img = L.n_img;
    std::vector<int32_t> nreg((size_t)n_img), r_off((size_t)n_img + 1, 0);
    CK(ctx, cudaMemcpyAsync(nreg.data(), L.n_regions, (size_t)n_img * 4, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    for (int i = 0; i < n_img; ++i) r_off[(size_t)i + 1] = r_off[(size_t)i] + nreg[(size_t)i];
    const size_t R = (size_t)r_off[(size_t)n_img];
    std::vector<LsdRegion> regs(R);
    for (int i = 0; i < n_img; ++i)
        if (nreg[(size_t)i])
            CK(ctx, cudaMemcpyAsync(regs.data() + r_off[(size_t)i], L.regions + (size_t)i * L.reg_cap,
                                    (size_t)nreg[(size_t)i] * sizeof(LsdRegion), cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    std::vector<double2> dir(R);
    for (size_t r = 0; r < R; ++r) dir[r] = make_double2(cos(regs[r].theta), sin(regs[r].theta));
    Arena b;
    const size_t o_roff = b.take(((size_t)n_img + 1) * 4), o_dir = b.take(R * 16), o_seg = b.take(R * 16);
    CK(ctx, b.alloc(ctx->arena_lsd_seg));
    CK(ctx, b.up(o_roff, r_off.data(), ((size_t)n_img + 1) * 4, s));
    CK(ctx, b.up(o_dir, dir.data(), R * 16, s));
    cudaEvent_t* ev = ctx->lsd_ev.ev;
    int launches = 0;
    CK(ctx, cudaEventRecord(ev[4], s));
    CK(ctx, launch_lsd_extent(L, (int)R, b.i32(o_roff), b.at<double2>(o_dir), b.at<float4>(o_seg), s, &launches));
    CK(ctx, cudaEventRecord(ev[5], s));
    ctx->lsd_ran = true;
    ctx->launches += launches;
    std::vector<float4> raw(R);
    CK(ctx, b.down(raw.data(), o_seg, R * 16, s));
    CK(ctx, cudaStreamSynchronize(s));
    const double min_length = cfg->min_line_length * std::min(L.W, L.H);
    kls.assign((size_t)n_img, {});
    for (int i = 0; i < n_img; ++i)
        lsd_keylines(L.W, L.H, raw.data() + r_off[(size_t)i], nreg[(size_t)i], min_length, cfg->n_features, kls[(size_t)i]);
    return 0;
}

// the key lines of images i0 .. i0 + n - 1 as rows from row 0 of each array (a null array is skipped)
void lsd_rows(const std::vector<std::vector<KeyLine>>& kls, int i0, int n, float* seg, float* angle, int32_t* npix,
              float* response, float* length) {
    size_t r = 0;
    for (int i = i0; i < i0 + n; ++i)
        for (const KeyLine& kl : kls[(size_t)i]) {
            if (seg) memcpy(seg + 4 * r, kl.seg, sizeof kl.seg);
            if (angle) angle[r] = kl.angle;
            if (npix) npix[r] = kl.npix;
            if (response) response[r] = kl.response;
            if (length) length[r] = kl.length;
            ++r;
        }
}
}  // namespace

int plstvo_lsd_detect_batch(PlContext* ctx, const PlLsdConfig* cfg, int n_img, int width, int height, const uint8_t* images,
                            int capacity, int32_t* kl_off, float* kl_seg, float* kl_angle, int32_t* kl_npix,
                            float* kl_response, float* kl_length) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!cfg || n_img < 0 || capacity < 0) return fail(ctx, PLSTVO_E_INVALID, "null config, negative n_img or negative capacity");
    if (n_img > 65535) return fail(ctx, PLSTVO_E_INVALID, "more than 65535 images in one call");   // gridDim.z of the pixel kernels
    if (width < 1 || width > 32767 || height < 1 || height > 32767) return fail(ctx, PLSTVO_E_INVALID, "width and height must be 1..32767");
    if (const int rc = lsd_check_config(ctx, cfg)) return rc;
    if (!kl_off) return fail(ctx, PLSTVO_E_INVALID, "null kl_off");
    LsdLaunch L;
    if (const int rc = lsd_plan(ctx, cfg, n_img, width, height, L)) return rc;
    kl_off[0] = 0;
    if (n_img == 0) return 0;
    if (!images) return fail(ctx, PLSTVO_E_INVALID, "null images");
    if (const int rc = lsd_enqueue(ctx, L, nullptr, nullptr, {ImgPart{images, n_img}}, ctx->s_main)) return rc;
    std::vector<std::vector<KeyLine>> kls;
    if (const int rc = lsd_finish(ctx, cfg, L, ctx->s_main, kls)) return rc;
    // kl_off in full before any capacity check
    bool too_many = false;
    for (int i = 0; i < n_img; ++i) {
        const long next = (long)kl_off[i] + (long)kls[(size_t)i].size();
        too_many |= kls[(size_t)i].size() > (size_t)PLSTVO_MAX_FEATURES || next > INT_MAX;
        kl_off[i + 1] = (int32_t)std::min(next, (long)INT_MAX);
    }
    if (too_many) return fail(ctx, PLSTVO_E_TOO_LARGE, "more than 65535 key lines in one image");
    if (kl_off[n_img] > capacity) return fail(ctx, PLSTVO_E_TOO_LARGE, "more key lines than capacity");
    lsd_rows(kls, 0, n_img, kl_seg, kl_angle, kl_npix, kl_response, kl_length);
    return kl_off[n_img];
}

int plstvo_lsd_kernel_times(PlContext* ctx, float* ms5) {
    if (!ctx || !ms5) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!ctx->lsd_ran) return fail(ctx, PLSTVO_E_INVALID, "no LSD call on this context yet");
    CK(ctx, cudaSetDevice(ctx->device));
    for (int k = 0; k < 5; ++k) CK(ctx, cudaEventElapsedTime(&ms5[k], ctx->lsd_ev[k], ctx->lsd_ev[k + 1]));
    return 0;
}

int plstvo_fld_key_lines(int width, int height, int n_features, int n_seg, const float* seg, float* kl_seg, float* kl_angle,
                         int32_t* kl_npix, float* kl_response, float* kl_length) {
    if (width < 1 || width > 32767 || height < 1 || height > 32767 || n_features < 0 || n_seg < 0 || (n_seg && !seg))
        return PLSTVO_E_INVALID;
    // LineIterator rounds with cvRound, which equals lrintf only on finite values inside int (it gives INT_MIN elsewhere), and
    // the sort needs ordered lengths: such coordinates are refused rather than counted differently
    for (size_t k = 0; k < 4 * (size_t)n_seg; ++k)
        if (!(seg[k] >= -2147483648.0f && seg[k] < 2147483648.0f)) return PLSTVO_E_INVALID;
    std::vector<KeyLine> kls;
    fld_keylines(width, height, seg, n_seg, n_features, kls);
    const std::vector<std::vector<KeyLine>> one{std::move(kls)};
    lsd_rows(one, 0, 1, kl_seg, kl_angle, kl_npix, kl_response, kl_length);
    return (int)one[0].size();
}

/* ---- stereo images -> pose: ORB, LSD and LBD feed the stereo step and the tracker without leaving HBM ---- */
namespace {
// A call's key lines in blocks of nf images, block 2 s + side holding step (or frame set) s's left (side 0) or right images:
// the LineSrc each block gives LBD and the stereo step, and where LBD leaves the blocks' rows
struct LineBlocks {
    std::vector<LineSrc> lsrc;                     // per block: into the caller's arrays, or into LSD's below
    std::vector<std::vector<int32_t>> off;         // per block: its offsets, rebased to 0
    std::vector<int32_t> lsd_off, lsd_npix;        // LSD's key lines of every image of the call
    std::vector<float> lsd_seg, lsd_angle;
    std::vector<int32_t> lbase{0};                 // [blocks + 1] each block's first row in LBD's output
    bool run_lbd = false;                          // some block has a key line
    const float* d_seg = nullptr;                  // LBD's rows (once describe() ran): segments and descriptors
    const uint8_t* d_ldesc = nullptr;
    cudaEvent_t joined = nullptr;                  // recorded on the second stream after LBD

    // The caller's key lines of frame sets fs[0 .. nfs), steps x nf frames each: both sides of every set checked whole, then
    // cut into one block per step and side
    int cut(PlContext* ctx, const PlStereoImages* const* fs, int nfs, int steps, int nf) {
        std::vector<LineSrc> whole;
        for (int j = 0; j < nfs; ++j) {
            whole.push_back(LineSrc{steps * nf, fs[j]->ll_off, fs[j]->seg_l, fs[j]->angle_l, fs[j]->npix_l});
            whole.push_back(LineSrc{steps * nf, fs[j]->lr_off, fs[j]->seg_r, fs[j]->angle_r, fs[j]->npix_r});
        }
        for (const LineSrc& l : whole)
            if (const int rc = lbd_check_lines(ctx, l)) return rc;
        off.assign(whole.size() * steps, {});
        for (size_t b = 0; b < off.size(); ++b)   // frame set b / (2 steps), step b / 2 % steps, side b % 2
            add_block(b, whole[b / (2 * steps) * 2 + b % 2], b / 2 % steps * nf, nf);
        return 0;
    }

    // The caller's key lines of f's B frames, both sides checked whole, then one block per image in the order the call's
    // images took on the device: block z is image side[z] (0 left, 1 right) of frame frame[z]
    int cut_images(PlContext* ctx, const PlStereoImages* f, const std::vector<int>& frame, const std::vector<int>& side) {
        const LineSrc whole[2] = {LineSrc{f->B, f->ll_off, f->seg_l, f->angle_l, f->npix_l},
                                  LineSrc{f->B, f->lr_off, f->seg_r, f->angle_r, f->npix_r}};
        for (const LineSrc& l : whole)
            if (const int rc = lbd_check_lines(ctx, l)) return rc;
        off.assign(frame.size(), {});
        for (size_t z = 0; z < frame.size(); ++z) add_block(z, whole[side[z]], (size_t)frame[z], 1);
        return 0;
    }

    // LSD's key lines of nblk blocks of nf images: its host continuation on stream s (where its device half ran), with the
    // images calls' key-line checks
    int take_lsd(PlContext* ctx, const PlLsdConfig* lc, const LsdLaunch& lsd, cudaStream_t s, int nblk, int nf) {
        std::vector<std::vector<KeyLine>> kls;
        if (const int rc = lsd_finish(ctx, lc, lsd, s, kls)) return rc;
        lsd_off.assign(1, 0);
        for (const std::vector<KeyLine>& k : kls) {
            if (k.size() > (size_t)PLSTVO_MAX_FEATURES) return fail(ctx, PLSTVO_E_TOO_LARGE, "more than 65535 key lines in one image");
            lsd_off.push_back(lsd_off.back() + (int32_t)k.size());
        }
        const size_t m = (size_t)lsd_off.back();
        lsd_seg.resize(4 * m);
        lsd_angle.resize(m);
        lsd_npix.resize(m);
        lsd_rows(kls, 0, (int)kls.size(), lsd_seg.data(), lsd_angle.data(), lsd_npix.data(), nullptr, nullptr);
        const LineSrc all{(int)kls.size(), lsd_off.data(), lsd_seg.data(), lsd_angle.data(), lsd_npix.data()};
        if (const int rc = lbd_check_lines(ctx, all)) return rc;
        off.assign((size_t)nblk, {});
        for (int b = 0; b < nblk; ++b) add_block(b, all, (size_t)b * nf, nf);
        return 0;
    }

    // block b (the next one): nf images of l from image i0 on
    void add_block(size_t b, const LineSrc& l, size_t i0, int nf) {
        const int32_t* o = l.off + i0;
        for (int i = 0; i <= nf; ++i) off[b].push_back(o[i] - o[0]);
        lsrc.push_back(LineSrc{nf, off[b].data(), l.seg + 4 * (size_t)o[0], l.angle + o[0], l.npix + o[0]});
        lbase.push_back(lbase.back() + off[b][(size_t)nf]);
        run_lbd = lbase.back() > 0;
    }

    // LBD on every block's key lines, enqueued on the second stream (device images d_img, ready once `ready` has completed,
    // or host images parts), then the join
    int describe(PlContext* ctx, int W, int H, const uint8_t* d_img, cudaEvent_t ready, const std::vector<ImgPart>& parts) {
        if (const int rc = lbd_enqueue(ctx, W, H, lsrc, d_img, ready, parts, ctx->s_alt, &d_seg, &d_ldesc)) return rc;
        CK(ctx, cudaEventRecord(ctx->img_join[0], ctx->s_alt));
        joined = ctx->img_join[0];
        return 0;
    }
};

// One frame set of the stereo step (nf frames) on device inputs, into fs[0] (points) and fs[1] (lines): the points of ORB's
// image blocks ob and ob + 1 (left, right, nf images each) and the key lines of line blocks lb and lb + 1, offsets rebased to
// 0 into pl_off / pr_off.  none: nf + 1 zero offsets, for frames without key lines.
void stereo_set_inputs(const OrbDetected& orb, int ob, bool pts, const LineBlocks& lines, int lb, int nf,
                       const std::vector<int32_t>& none, std::vector<int32_t>& pl_off, std::vector<int32_t>& pr_off,
                       StereoSet* fs) {
    const size_t kl = orb.off[(size_t)ob * nf], kr = orb.off[(size_t)(ob + 1) * nf];
    pl_off.resize((size_t)nf + 1);
    pr_off.resize((size_t)nf + 1);
    for (int i = 0; i <= nf; ++i) {
        pl_off[i] = orb.off[(size_t)ob * nf + i] - (int32_t)kl;
        pr_off[i] = orb.off[(size_t)(ob + 1) * nf + i] - (int32_t)kr;
    }
    StereoSet& P = fs[0];
    P = StereoSet{false, nf, pl_off.data(), pr_off.data(), nullptr, true};
    if (pts) {
        P.xy_l = orb.xy + 2 * kl; P.xy_r = orb.xy + 2 * kr; P.oct = orb.octave + kl;
        P.d1 = orb.desc + 32 * kl; P.d2 = orb.desc + 32 * kr;
    }
    StereoSet& Ls = fs[1];   // oct stays null: key lines of octave 0
    Ls = StereoSet{true, nf, none.data(), none.data(), nullptr, true};
    if (!lines.lsrc.empty()) {
        Ls.l_off = lines.lsrc[(size_t)lb].off; Ls.r_off = lines.lsrc[(size_t)lb + 1].off; Ls.ang = lines.lsrc[(size_t)lb].angle;
    }
    if (lines.run_lbd) {
        const size_t l0 = (size_t)lines.lbase[(size_t)lb], l1 = (size_t)lines.lbase[(size_t)lb + 1];
        Ls.xy_l = lines.d_seg + 4 * l0; Ls.xy_r = lines.d_seg + 4 * l1;
        Ls.d1 = lines.d_ldesc + 32 * l0; Ls.d2 = lines.d_ldesc + 32 * l1;
    }
}

// The line set of one group of a scheduled run (nf frames): line blocks of one image each, lb .. lb + nf - 1 the left images
// and the next nf the right ones.  Their offsets and left angles are joined into l_off, r_off and ang (host), and the rows
// are one slice of LBD's output, as the blocks are consecutive.
void schedule_line_inputs(const LineBlocks& lines, int lb, int nf, std::vector<int32_t>& l_off, std::vector<int32_t>& r_off,
                          std::vector<float>& ang, StereoSet& Ls) {
    if (lines.lsrc.empty()) return;
    l_off.assign(1, 0);
    r_off.assign(1, 0);
    ang.clear();
    for (int i = 0; i < nf; ++i) {
        const LineSrc& l = lines.lsrc[(size_t)lb + i];
        const LineSrc& r = lines.lsrc[(size_t)(lb + nf + i)];
        l_off.push_back(l_off.back() + l.off[1]);
        r_off.push_back(r_off.back() + r.off[1]);
        ang.insert(ang.end(), l.angle, l.angle + l.off[1]);
    }
    Ls.l_off = l_off.data();
    Ls.r_off = r_off.data();
    Ls.ang = ang.data();
    if (lines.run_lbd) {
        const size_t l0 = (size_t)lines.lbase[(size_t)lb], l1 = (size_t)lines.lbase[(size_t)(lb + nf)];
        Ls.xy_l = lines.d_seg + 4 * l0; Ls.xy_r = lines.d_seg + 4 * l1;
        Ls.d1 = lines.d_ldesc + 32 * l0; Ls.d2 = lines.d_ldesc + 32 * l1;
    }
}

// The key-line field rules of a call on frame sets fs[0 .. nfs): the fields are null where the call detects its own key lines
// (detect) and in a session without lines (no_lines); a session run (run) sets its own FAST thresholds, so frames->fast_th is
// null there too
int check_key_line_fields(PlContext* ctx, const PlStereoImages* const* fs, int nfs, bool detect, bool no_lines, bool run) {
    bool given = false;
    for (int j = 0; j < nfs; ++j) {
        const PlStereoImages* f = fs[j];
        given = given || f->ll_off || f->lr_off || f->seg_l || f->seg_r || f->angle_l || f->angle_r || f->npix_l || f->npix_r;
    }
    if (run && (fs[0]->fast_th || (detect && given)))
        return fail(ctx, PLSTVO_E_INVALID,
                    detect ? "frames->fast_th and the key-line fields must be null: the run sets its thresholds and detects its key lines"
                           : "frames->fast_th must be null: the run sets its thresholds");
    if (given && detect) return fail(ctx, PLSTVO_E_INVALID, "key-line fields must be null: the call detects its own key lines");
    if (given && no_lines) return fail(ctx, PLSTVO_E_INVALID, "key-line fields must be null: the session has no lines");
    return 0;
}

// The image checks of an images call or a session run, before any work, on frame sets fs[0 .. nfs) holding n_img > 0 images
// in all: every image of the camera's size and present where a stage runs, and with lines the size range and, given lc, LSD's
// plan of all n_img images
int images_check(PlContext* ctx, int W, int H, bool pts, bool lns, const PlStereoImages* const* fs, int nfs,
                 const PlLsdConfig* lc, int n_img, LsdLaunch& lsd) {
    for (int j = 0; j < nfs; ++j) {
        // the reference's grid scale is cols / img.cols (src/stereoFrame.cpp:47-48), the stereo step's cols / cam->width
        if (fs[j]->width != W || fs[j]->height != H) return fail(ctx, PLSTVO_E_SIZE, "image size differs from the camera's");
        if ((pts || lns) && (!fs[j]->img_l || !fs[j]->img_r)) return fail(ctx, PLSTVO_E_INVALID, "null images");
    }
    if (lns) {
        if (W < 1 || W > 32767 || H < 1 || H > 32767) return fail(ctx, PLSTVO_E_INVALID, "width and height must be 1..32767");
        if (lc)
            if (const int rc = lsd_plan(ctx, lc, n_img, W, H, lsd)) return rc;
    }
    return 0;
}

// Enqueues on s the grey device copy of n_img raw images (parts) in blocks of n images alternating left, right: the remap /
// colour conversion of rect, or in a session call with per-stream rectifiers, stream ids[k]'s rectifier for image k of each
// block.  A colour session on the FLD branch with lines also gets the RGB2GRAY plane LBD reads (*d_lbd; else null).
int rectify_call(PlContext* ctx, const PlRectifier* rect, const SessionCall* call, int n, int n_img,
                 const std::vector<ImgPart>& parts, cudaStream_t s, const uint8_t** d_out, const uint8_t** d_lbd) {
    const PlStereoSession* ss = call ? call->ss : nullptr;
    std::vector<const PlRectifier*> call_rects;   // a session's per-stream rectifiers, call order
    if (ss && !ss->rects.empty())
        for (int k = 0; k < n; ++k) call_rects.push_back(ss->rects[(size_t)call->ids[k]]);
    const bool rgb = ss && ss->fld && ss->cfg.has_lines && rect->channels > 1;
    return rectify_enqueue(ctx, rect, n_img, n, parts, s, d_out, call_rects.empty() ? nullptr : call_rects.data(),
                           rgb ? d_lbd : nullptr);
}
}  // namespace

// The images go up once, in blocks of NF images: sequence [left][right], batch [prev left][prev right][curr left][curr right].
// Every feature set of the stereo step is then a contiguous slice of ORB's CSR output and of LBD's rows.  The key lines are
// the caller's, or (detect_lines) LSD's, detected on the same device copy of the images: ORB's, or LSD's own when ORB does
// not run.  With a rectifier (raw images), that copy is the remap's output and every stage reads it.
static int track_images_run(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                            const PlStereoConfig* sc, const PlOrbDetectConfig* oc, bool detect_lines, const PlLsdConfig* lc,
                            const PlRectifier* rect, const PlStereoImages* prev, const PlStereoImages* curr,
                            const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo, bool sequence,
                            SessionCall* call = nullptr) {
    const bool one_set = sequence || call;   // one frame set: a sequence, or a session's new frames
    if (!cam || !cfg || !mc || !sc || !oc || !prev || (!one_set && !curr) || (!results && (!call || call->track)))
        return fail(ctx, PLSTVO_E_INVALID, "null argument");
    if (rect && rect->ctx != ctx) return fail(ctx, PLSTVO_E_INVALID, "the rectifier belongs to another context");
    if (rect && (rect->width != cam->width || rect->height != cam->height))
        return fail(ctx, PLSTVO_E_SIZE, "rectifier size differs from the camera's");
    const int NF = prev->B;
    if (NF < 0) return fail(ctx, PLSTVO_E_INVALID, "negative number of frames");
    if (!one_set && curr->B != NF) return fail(ctx, PLSTVO_E_SIZE, "prev and curr hold different numbers of frames");
    if (const int rc = orb_detect_check(ctx, oc)) return rc;
    const int nfs = one_set ? 1 : 2;   // frame sets: the sequence or the session's new frames, or prev and curr
    const PlStereoImages* fs[2] = {prev, curr};
    const bool pts = cfg->has_points != 0, lns = cfg->has_lines != 0, run_lsd = detect_lines && lns;
    const int W = cam->width, H = cam->height;
    if (const int rc = check_key_line_fields(ctx, fs, nfs, detect_lines, false, false)) return rc;
    if (run_lsd) {
        if (!lc) return fail(ctx, PLSTVO_E_INVALID, "null lsd config");
        if (const int rc = lsd_check_config(ctx, lc)) return rc;
        if (2L * nfs * NF > 65535) return fail(ctx, PLSTVO_E_INVALID, "more than 65535 images in one call");
    }
    const int nblk = 2 * nfs, n_img = nblk * NF;
    LineBlocks lines;   // key lines per image block: one frame set's left, right images
    LsdLaunch lsd{};
    if (NF > 0) {
        if (const int rc = images_check(ctx, W, H, pts, lns, fs, nfs, run_lsd ? lc : nullptr, n_img, lsd)) return rc;
        if (lns && !run_lsd)
            if (const int rc = lines.cut(ctx, fs, nfs, 1, NF)) return rc;
    }
    if (NF == 0 || (sequence && NF == 1)) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, ctx->img_ev.create());
    CK(ctx, ctx->img_join.create(cudaEventDisableTiming));
    ctx->img_timed = false;
    std::vector<ImgPart> iparts;
    std::vector<int32_t> th((size_t)n_img);
    for (int b = 0; b < nblk; ++b) {
        const PlStereoImages* f = fs[b / 2];
        iparts.push_back(ImgPart{b % 2 ? f->img_r : f->img_l, NF});
        for (int i = 0; i < NF; ++i)   // 0 = the configured threshold, as detectPointFeatures / plstvo::detectAndComputeORB
            th[(size_t)b * NF + i] = f->fast_th && f->fast_th[i] ? f->fast_th[i] : oc->fast_threshold;
    }
    // the host images a stage may upload itself: none with a rectifier, whose images (colour ones too) only the rectifier
    // reads; every stage then reads its grey device copy
    const std::vector<ImgPart> no_parts;
    const std::vector<ImgPart>& stage_parts = rect ? no_parts : iparts;
    const uint8_t* d_images = nullptr;   // the device copy of the images the line stages read (null: LBD uploads its own)
    const uint8_t* d_rgb = nullptr;      // a colour FLD session's RGB2GRAY plane, which LBD reads instead
    cudaEvent_t images_ready = nullptr;
    auto enqueue_lbd = [&]() { return lines.describe(ctx, W, H, d_rgb ? d_rgb : d_images, images_ready, stage_parts); };
    // With fewer images than SMs, LSD's one-warp and one-thread-per-image stages (seed order, region growing) are the whole
    // critical path and lose more beside ORB than ORB takes (BASELINE.md), so LSD runs first on the main stream, alone, and ORB
    // reads its device copy of the images; LBD then runs beside ORB as for the caller's key lines.  With more, ORB runs beside
    // LSD on the second stream.
    const bool lsd_first = run_lsd && pts && n_img < ctx->sm_count;
    CK(ctx, cudaEventRecord(ctx->img_ev[0], ctx->s_main));
    // raw images: they go up into the rectifier's staging slot, and every stage reads the grey device copy the rectifier
    // writes (the remap's, or for colour images the conversion's)
    const uint8_t* rectified = nullptr;
    cudaEvent_t rectified_ready = nullptr;
    if (rect && (pts || lns)) {
        if (const int rc = rectify_call(ctx, rect, call, NF, n_img, iparts, ctx->s_main, &rectified, &d_rgb))
            return rc;
        rectified_ready = next_event(ctx);
        CK(ctx, cudaEventRecord(rectified_ready, ctx->s_main));
    }
    const uint8_t* orb_images = rectified;   // the device images ORB reads (null: ORB uploads them)
    if (lsd_first) {
        if (const int rc = lsd_enqueue(ctx, lsd, rectified, nullptr, stage_parts, ctx->s_main)) return rc;
        if (const int rc = lines.take_lsd(ctx, lc, lsd, ctx->s_main, nblk, NF)) return rc;
        orb_images = lsd.images;
    }
    const bool lsd_beside = run_lsd && !lsd_first;
    // the line stage that runs on the second stream beside ORB: LSD's device half, or LBD on the caller's or LSD's key lines.
    // With ORB running it reads ORB's device images once they are there
    auto lines_beside = [&](const uint8_t* d_img, cudaEvent_t ready) -> int {
        d_images = d_img;
        images_ready = ready;
        return lsd_beside ? lsd_enqueue(ctx, lsd, d_img, ready, stage_parts, ctx->s_alt) : enqueue_lbd();
    };
    OrbDetected orb;
    if (pts) {
        std::function<int(const uint8_t*, cudaEvent_t)> beside;
        if (lsd_beside || lines.run_lbd) beside = lines_beside;
        if (const int rc = orb_detect_enqueue(ctx, oc, n_img, W, H, orb_images, stage_parts, th.data(), INT_MAX, beside, orb))
            return rc;
    } else {
        orb.off.assign((size_t)n_img + 1, 0);
        if (lsd_beside || lines.run_lbd)
            if (const int rc = lines_beside(rectified, rectified_ready)) return rc;
    }
    if (lsd_beside) {   // LSD's host continuation (while ORB's selection and descriptors run), then LBD on the same stream
        if (const int rc = lines.take_lsd(ctx, lc, lsd, ctx->s_alt, nblk, NF)) return rc;
        d_images = lsd.images;   // ORB's copy, or LSD's own when ORB does not run
        if (lines.run_lbd)
            if (const int rc = enqueue_lbd()) return rc;
    }
    // the feature sets: slices of ORB's and LBD's outputs, offsets rebased to 0
    std::vector<int32_t> pl_off[2], pr_off[2], none((size_t)NF + 1, 0);
    StereoSet sets[2][2];
    for (int j = 0; j < nfs; ++j) stereo_set_inputs(orb, 2 * j, pts, lines, 2 * j, NF, none, pl_off[j], pr_off[j], sets[j]);
    StereoDevInputs dev;
    dev.lines_ready = lines.joined;
    dev.marks = ctx->img_ev.ev + 1;
    if (const int rc = track_stereo_common(ctx, cam, cfg, mc, sc, sets[0], one_set ? nullptr : sets[1], priors, results,
                                           n_stereo, sequence, -1, &dev, call))
        return rc;
    float* ms = ctx->img_ms;   // the call ended synchronised: every event has completed
    std::fill(ms, ms + 5, 0.f);
    // uploads end where the first stage starts: LSD waits for the images, LBD on the caller's lines for the images and its key
    // lines, ORB for the images only
    const bool run_lbd = lines.run_lbd;
    const cudaEvent_t up_end = run_lsd ? ctx->lsd_ev[0] : run_lbd ? ctx->lbd_ev[0] : pts ? ctx->orb_det_ev[0] : nullptr;
    if (up_end) CK(ctx, cudaEventElapsedTime(&ms[0], ctx->img_ev[0], up_end));
    if (pts) CK(ctx, cudaEventElapsedTime(&ms[1], ctx->orb_det_ev[0], ctx->orb_det_ev[4]));
    // the lines: LSD's first launch (host hops included) to LBD's last, or LBD alone on the caller's lines
    if (run_lsd || run_lbd)
        CK(ctx, cudaEventElapsedTime(&ms[2], run_lsd ? ctx->lsd_ev[0] : ctx->lbd_ev[0], run_lbd ? ctx->lbd_ev[2] : ctx->lsd_ev[5]));
    CK(ctx, cudaEventElapsedTime(&ms[3], ctx->img_ev[1], ctx->img_ev[2]));
    CK(ctx, cudaEventElapsedTime(&ms[4], ctx->img_ev[2], ctx->img_ev[3]));
    ctx->img_timed = true;
    return 0;
}

static int track_images_common(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                               const PlStereoConfig* sc, const PlOrbDetectConfig* oc, bool detect_lines, const PlLsdConfig* lc,
                               const PlStereoImages* prev, const PlStereoImages* curr, const PlPrior* priors,
                               PlPoseResult* results, int32_t* n_stereo, bool sequence, const PlRectifier* rect = nullptr,
                               SessionCall* call = nullptr) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    const int rc = track_images_run(ctx, cam, cfg, mc, sc, oc, detect_lines, lc, rect, prev, curr, priors, results, n_stereo,
                                    sequence, call);
    // after an error the line stages may still run on the second stream, and ORB on the first: the next call may reuse their
    // arenas
    const cudaError_t e = cudaStreamSynchronize(ctx->s_alt), e_main = cudaStreamSynchronize(ctx->s_main);
    if (rc) return rc;
    CK(ctx, e);
    CK(ctx, e_main);
    return 0;
}

int plstvo_track_stereo_images_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                     const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlStereoImages* prev,
                                     const PlStereoImages* curr, const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    return track_images_common(ctx, cam, cfg, mcfg, scfg, ocfg, false, nullptr, prev, curr, priors, results, n_stereo, false);
}

int plstvo_track_stereo_images_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                        const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlStereoImages* frames,
                                        const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    return track_images_common(ctx, cam, cfg, mcfg, scfg, ocfg, false, nullptr, frames, nullptr, priors, results, n_stereo, true);
}

int plstvo_track_stereo_images_lsd_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                         const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg,
                                         const PlStereoImages* prev, const PlStereoImages* curr, const PlPrior* priors,
                                         PlPoseResult* results, int32_t* n_stereo) {
    return track_images_common(ctx, cam, cfg, mcfg, scfg, ocfg, true, lcfg, prev, curr, priors, results, n_stereo, false);
}

int plstvo_track_stereo_images_lsd_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                                            const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                            const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg, const PlStereoImages* frames,
                                            const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    return track_images_common(ctx, cam, cfg, mcfg, scfg, ocfg, true, lcfg, frames, nullptr, priors, results, n_stereo, true);
}

int plstvo_track_stereo_raw_images_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mcfg,
                                         const PlStereoConfig* scfg, const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg,
                                         const PlRectifier* rect, const PlStereoImages* prev, const PlStereoImages* curr,
                                         const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    return track_images_common(ctx, cam, cfg, mcfg, scfg, ocfg, true, lcfg, prev, curr, priors, results, n_stereo, false, rect);
}

int plstvo_track_stereo_raw_images_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                                            const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                            const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg, const PlRectifier* rect,
                                            const PlStereoImages* frames, const PlPrior* priors, PlPoseResult* results,
                                            int32_t* n_stereo) {
    return track_images_common(ctx, cam, cfg, mcfg, scfg, ocfg, true, lcfg, frames, nullptr, priors, results, n_stereo, true, rect);
}

/* ---- stereo sessions: each stream's previous frame kept in HBM as its stereo features ---- */
PlStereoSession* plstvo_stereo_session_create(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg,
                                              const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                              const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg, const PlRectifier* rect,
                                              int n_streams) {
    if (!ctx) return nullptr;
    LOCK(ctx);
    auto bad = [&](int code, const char* msg) -> PlStereoSession* {
        fail(ctx, code, msg);
        return nullptr;
    };
    if (!cam || !cfg || !mcfg || !scfg || !ocfg) return bad(PLSTVO_E_INVALID, "null argument");
    if (n_streams < 1) return bad(PLSTVO_E_INVALID, "n_streams must be at least 1");
    if (orb_detect_check(ctx, ocfg)) return nullptr;
    if (cfg->has_lines) {
        if (!lcfg) return bad(PLSTVO_E_INVALID, "null lsd config");
        if (lsd_check_config(ctx, lcfg)) return nullptr;
    }
    if (!grid_ok(mcfg->grid_rows, mcfg->grid_cols) || cam->width <= 0 || cam->height <= 0)
        return bad(PLSTVO_E_INVALID, "bad grid or image size");
    if (rect && rect->ctx != ctx) return bad(PLSTVO_E_INVALID, "the rectifier belongs to another context");
    if (rect && (rect->width != cam->width || rect->height != cam->height))
        return bad(PLSTVO_E_SIZE, "rectifier size differs from the camera's");
    PlStereoSession* ss = new PlStereoSession();
    ss->ctx = ctx;
    ss->cam = *cam; ss->cfg = *cfg; ss->mc = *mcfg; ss->sc = *scfg; ss->oc = *ocfg;
    ss->has_lc = lcfg != nullptr;
    if (lcfg) ss->lc = *lcfg;
    ss->rect = rect;
    ss->n_streams = n_streams;
    ss->live.assign((size_t)n_streams, 0);
    ss->n_pt.assign((size_t)n_streams, 0);
    ss->n_ls.assign((size_t)n_streams, 0);
    ss->off_pt.assign((size_t)n_streams, 0);
    ss->off_ls.assign((size_t)n_streams, 0);
    return ss;
}

PlStereoSession* plstvo_stereo_session_create_cams(PlContext* ctx, const PlCamera* cams, const PlConfig* cfg,
                                                   const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                                                   const PlOrbDetectConfig* ocfg, const PlLsdConfig* lcfg,
                                                   const PlRectifier* const* rects, int n_streams) {
    if (!ctx) return nullptr;
    LOCK(ctx);
    auto bad = [&](int code, const char* msg) -> PlStereoSession* {
        fail(ctx, code, msg);
        return nullptr;
    };
    if (!cams) return bad(PLSTVO_E_INVALID, "null cameras");
    if (n_streams < 1) return bad(PLSTVO_E_INVALID, "n_streams must be at least 1");
    for (int i = 1; i < n_streams; ++i)
        if (cams[i].width != cams[0].width || cams[i].height != cams[0].height)
            return bad(PLSTVO_E_SIZE, "the cameras differ in image size");
    // the rectifier the images path sizes its staging by (the first one given), after every entry is checked against it
    const PlRectifier* first = nullptr;
    bool any_null = false;
    for (int i = 0; rects && i < n_streams; ++i) {
        const PlRectifier* r = rects[i];
        if (!r) {
            any_null = true;
            continue;
        }
        if (r->ctx != ctx) return bad(PLSTVO_E_INVALID, "a rectifier belongs to another context");
        if (r->width != cams[0].width || r->height != cams[0].height)
            return bad(PLSTVO_E_SIZE, "rectifier size differs from the cameras'");
        if (first && r->channels != first->channels) return bad(PLSTVO_E_INVALID, "the rectifiers differ in channel count");
        if (!first) first = r;
    }
    if (first && first->channels > 1 && any_null)
        return bad(PLSTVO_E_INVALID, "a colour session needs a colour rectifier for every stream (one without maps converts only)");
    PlStereoSession* ss = plstvo_stereo_session_create(ctx, &cams[0], cfg, mcfg, scfg, ocfg, lcfg, first, n_streams);
    if (!ss) return nullptr;
    ss->cams.assign(cams, cams + n_streams);
    if (first) ss->rects.assign(rects, rects + n_streams);   // all null: no stream is remapped, as with rects == NULL
    return ss;
}

void plstvo_stereo_session_destroy(PlStereoSession* ss) {
    if (!ss) return;
    {
        LOCK(ss->ctx);   // every call that reads the pools blocks, so none is using them once the lock is held
        cudaSetDevice(ss->ctx->device);
        ss->pool[0].buf.release();
        ss->pool[1].buf.release();
        ss->d_meta.release();
        ss->kept.buf.release();
        ss->d_cams.release();
        ss->kf_steps.clear();
    }
    delete ss;
}

int64_t plstvo_stereo_session_device_bytes(const PlStereoSession* ss) {
    if (!ss) return 0;
    LOCK(ss->ctx);
    size_t kf = 0;
    for (const auto& c : ss->kf_steps) kf += c->buf.cap;
    return (int64_t)(ss->pool[0].buf.cap + ss->pool[1].buf.cap + ss->d_meta.cap + ss->kept.buf.cap + ss->d_cams.cap + kf);
}

namespace {
// every session entry point, after the context lock: a session of this context (a read passes ss null where its output is
// null, with its own message)
int session_check(PlContext* ctx, const PlStereoSession* ss, const char* null_msg = "null session") {
    if (!ss) return fail(ctx, PLSTVO_E_INVALID, null_msg);
    if (ss->ctx != ctx) return fail(ctx, PLSTVO_E_INVALID, "the session belongs to another context");
    return 0;
}

// every call on a session but the reads discards the key frames a run_keyframes kept (the chunks' frees wait for the device)
void session_drop_keyframes(PlStereoSession* ss) {
    ss->kf_valid = false;
    if (!ss->kf_steps.empty()) cudaSetDevice(ss->ctx->device);
    ss->kf_steps.clear();
    ss->kf_rows.clear();
    ss->kf_off.clear();
}

// The start and the end of a call that changes the session: initialize / insert, run and run_keyframes.  The start drops the
// key frames and, with discard, invalidates what the last call retained.  The end of a failed call (rc) does both and
// synchronises both streams: the line stages may still run on the second stream, and ORB or a step on the first, and the
// next call may reuse their arenas.  The end of a successful one marks the retention arena as the call's (track, n): an empty
// call (n = 0) retains nothing, and a run of T = 0 (ran false) leaves it as it was.
void session_start(PlStereoSession* ss, bool discard) {
    if (discard) ss->kept.valid = false;
    session_drop_keyframes(ss);
}

int session_finish(PlContext* ctx, PlStereoSession* ss, int rc, bool track, int n, bool ran = true) {
    if (rc) {
        ss->kept.valid = false;
        session_drop_keyframes(ss);
        cudaStreamSynchronize(ctx->s_alt);
        cudaStreamSynchronize(ctx->s_main);
        return rc;
    }
    if (ran && ss->retain) {
        ss->kept.track = track;
        ss->kept.n = n;
        ss->kept.valid = n > 0 || ss->kept.lay_out(0, 0, 0, 0) == cudaSuccess;
    }
    return 0;
}

// the caller's arrays of a PlStereoFrameOut, indexed by records.h's arrays
RecPtrs frame_out_records(const PlStereoFrameOut* o) {
    return RecPtrs::from(PT_PL, {o->pt_pl, o->pt_disp, o->pt_P, o->pt_sigma2, o->pt_level, o->pdesc, o->pt_src,
                                 o->ls_spl, o->ls_epl, o->ls_sdisp, o->ls_edisp, o->ls_sP, o->ls_eP, o->ls_le, o->ls_angle,
                                 o->ls_sigma2, o->ls_level, o->ldesc, o->ls_src, o->m12_pt, o->inlier_pt, o->m12_ls,
                                 o->inlier_ls});
}
}  // namespace

int plstvo_stereo_session_retain(PlContext* ctx, PlStereoSession* ss, int on) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, ss)) return rc;
    if (on && ss->retain) return 0;   // already on: what the last call retained stays readable
    ss->retain = on != 0;
    session_drop_keyframes(ss);
    ss->kept.valid = false;
    if (!on) {
        CK(ctx, cudaSetDevice(ctx->device));
        ss->kept.buf.release();   // every call that wrote it blocked until done
    }
    return 0;
}

int plstvo_stereo_session_read(PlContext* ctx, const PlStereoSession* ss, const PlStereoFrameOut* out) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, out ? ss : nullptr, "null session or output")) return rc;
    if (!ss->retain) return fail(ctx, PLSTVO_E_INVALID, "retention is off: plstvo_stereo_session_retain(ctx, s, 1) first");
    const SessionRetained& kr = ss->kept;
    if (!kr.valid) return fail(ctx, PLSTVO_E_INVALID, "nothing retained: no call succeeded since retention was turned on, or the last call failed");
    CK(ctx, cudaSetDevice(ctx->device));
    const RecPtrs dst = frame_out_records(out);
    const int n_arrays = kr.track ? N_REC : M12_PT;   // after an initialize the tracker's arrays are left untouched
    cudaStream_t s = ctx->s_main;
    for (int k = 0; k < n_arrays; ++k) {
        const size_t bytes = kr.rows[k] * (size_t)REC_BYTES[k];
        if (dst.p[k] && bytes) CK(ctx, cudaMemcpyAsync(dst.p[k], kr.rec.p[k], bytes, cudaMemcpyDeviceToHost, s));
    }
    CK(ctx, cudaStreamSynchronize(s));
    return kr.n;
}

namespace {
// the named streams of a call: ids in range, no duplicates, and for an insert each holding a frame
int session_check_ids(PlContext* ctx, const PlStereoSession* ss, bool track, int n, const int32_t* ids) {
    std::vector<uint8_t> named((size_t)ss->n_streams, 0);
    for (int k = 0; k < n; ++k) {
        const int id = ids[k];
        if (id < 0 || id >= ss->n_streams) return fail(ctx, PLSTVO_E_INVALID, "stream id outside [0, n_streams)");
        if (named[(size_t)id]) return fail(ctx, PLSTVO_E_INVALID, "duplicate stream id");
        named[(size_t)id] = 1;
        if (track && !ss->live[(size_t)id]) return fail(ctx, PLSTVO_E_INVALID, "insert on a stream with no frame: initialize it first");
    }
    return 0;
}

// A call (or run step) on checked streams ids[0 .. n), filling the retention arena while retention is on; for an insert, the
// streams' kept frames compact in call order (the tracker's previous frames)
SessionCall session_begin(PlStereoSession* ss, bool track, int n, const int32_t* ids) {
    SessionCall c{ss, track, ss->retain, n, ids};
    if (!track) return c;
    c.kept_off_pt.assign((size_t)n + 1, 0);
    c.kept_off_ls.assign((size_t)n + 1, 0);
    for (int k = 0; k < n; ++k) {
        const size_t id = (size_t)ids[k];
        c.kept_off_pt[(size_t)k + 1] = c.kept_off_pt[(size_t)k] + ss->n_pt[id];
        c.kept_off_ls[(size_t)k + 1] = c.kept_off_ls[(size_t)k] + ss->n_ls[id];
    }
    return c;
}

// initialize (track == false) or insert for streams ids[0 .. n) after the session's start: the checks, then the images path
// with the call's record; the pools flip and the streams' counts are kept only when the whole call succeeded
int session_images(PlContext* ctx, PlStereoSession* ss, bool track, int n, const int32_t* ids, const PlStereoImages* frames,
                   const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    if (n < 0 || !frames) return fail(ctx, PLSTVO_E_INVALID, "null frames or negative n");
    if (frames->B != n) return fail(ctx, PLSTVO_E_SIZE, "frames->B differs from n");
    if (n == 0) return 0;
    if (!ids) return fail(ctx, PLSTVO_E_INVALID, "null ids");
    if (2L * n > 65535) return fail(ctx, PLSTVO_E_INVALID, "more than 65535 images in one call");
    if (const int rc = session_check_ids(ctx, ss, track, n, ids)) return rc;
    if (const int rc = check_key_line_fields(ctx, &frames, 1, false, ss->fld && !ss->cfg.has_lines, false)) return rc;
    SessionCall call = session_begin(ss, track, n, ids);
    // the FLD branch: the caller's key lines (the images call's checks), LSD and its config unused
    const int rc = track_images_common(ctx, &ss->cam, &ss->cfg, &ss->mc, &ss->sc, &ss->oc, !ss->fld,
                                       !ss->fld && ss->has_lc ? &ss->lc : nullptr, frames, nullptr, priors, results, n_stereo,
                                       false, ss->rect, &call);
    if (rc == 0) session_commit(call);
    return rc;
}

int session_call(PlContext* ctx, PlStereoSession* ss, bool track, int n, const int32_t* ids, const PlStereoImages* frames,
                 const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, ss)) return rc;
    session_start(ss, true);
    return session_finish(ctx, ss, session_images(ctx, ss, track, n, ids, frames, priors, results, n_stereo), track, n);
}
}  // namespace

int plstvo_stereo_session_initialize(PlContext* ctx, PlStereoSession* ss, int n, const int32_t* ids, const PlStereoImages* frames,
                                     int32_t* n_stereo) {
    return session_call(ctx, ss, false, n, ids, frames, nullptr, nullptr, n_stereo);
}

int plstvo_stereo_session_insert(PlContext* ctx, PlStereoSession* ss, int n, const int32_t* ids, const PlStereoImages* frames,
                                 const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    return session_call(ctx, ss, true, n, ids, frames, priors, results, n_stereo);
}

int plstvo_stereo_session_use_fld_lines(PlContext* ctx, PlStereoSession* ss, int on) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, ss)) return rc;
    for (uint8_t l : ss->live)
        if (l) return fail(ctx, PLSTVO_E_INVALID, "a stream holds a frame: switch the line branch before any stream is initialised");
    ss->fld = on != 0;
    return 0;
}

/* ---- stereo sessions: the handler's frame loop over T frames per stream in one call ---- */
void plstvo_default_handler_config(PlHandlerConfig* h) {
    if (!h) return;
    h->adaptative_fast = 1; h->fast_min_th = 5; h->fast_max_th = 50; h->fast_inc_th = 5; h->fast_feat_th = 50;
    h->fast_err_th = 0.5f;
}

void plstvo_kitti_handler_config(PlHandlerConfig* h) {
    if (!h) return;
    plstvo_default_handler_config(h);
    h->fast_min_th = 7; h->fast_max_th = 30;
}

namespace {
// the handler config's checks of a session run
int handler_check(PlContext* ctx, const PlHandlerConfig* h) {
    if (!h) return fail(ctx, PLSTVO_E_INVALID, "null handler config");
    if (h->fast_min_th < 1 || h->fast_min_th > h->fast_max_th || h->fast_max_th > 255 || h->fast_inc_th < 0 ||
        h->fast_feat_th < 0 || !std::isfinite(h->fast_err_th))
        return fail(ctx, PLSTVO_E_INVALID, "handler config out of range");
    return 0;
}

// the key-frame arguments' checks of a session run with the test (n streams)
int keyframe_check(PlContext* ctx, const PlKeyframeConfig* k, int n, const PlKeyframeState* kf_state, const PlKeyframeResult* kf) {
    if (!k || !kf_state || !kf) return fail(ctx, PLSTVO_E_INVALID, "null key-frame config, state or results");
    if (std::isnan(k->min_entropy_ratio) || std::isnan(k->max_kf_t_dist) || std::isnan(k->max_kf_r_dist))
        return fail(ctx, PLSTVO_E_INVALID, "NaN in the key-frame config");
    for (int i = 0; i < n; ++i)
        if ((kf_state[i].prev_f_iskf != 0 && kf_state[i].prev_f_iskf != 1) || kf_state[i].N_prevKF_currF < 0)
            return fail(ctx, PLSTVO_E_INVALID, "key-frame state with prev_f_iskf outside {0, 1} or a negative N_prevKF_currF");
    return 0;
}

// plstvo_stereo_session_run after the context lock: the checks, then the state-independent stages once over every image
// (upload, rectifier, LSD, LBD) and the steps (ORB at the device threshold row, the stereo step, tracking, the handler
// update), each committed to the session as an insert is.  session_finish synchronises both streams after a failure.  With kc
// (plstvo_stereo_session_run_keyframes) each step also runs the key-frame test from kf_state's streams and, with retention
// on, keeps every step's records and copies the key frames' into the session's chunks; kf_state is written on success only.
int session_run(PlContext* ctx, PlStereoSession* ss, const PlHandlerConfig* h, int n, const int32_t* ids, int T,
                const PlStereoImages* frames, const int32_t* fast_th0, const PlPrior* priors, PlPoseResult* results,
                int32_t* fast_th, int32_t* n_stereo, const PlKeyframeConfig* kc = nullptr, PlKeyframeState* kf_state = nullptr,
                PlKeyframeResult* kf = nullptr) {
    if (const int rc = handler_check(ctx, h)) return rc;
    if (T < 0) return fail(ctx, PLSTVO_E_INVALID, "negative T");
    if (n < 0 || !frames) return fail(ctx, PLSTVO_E_INVALID, "null frames or negative n");
    if ((long long)frames->B != (long long)T * n) return fail(ctx, PLSTVO_E_SIZE, "frames->B differs from T * n");
    const bool lns = ss->cfg.has_lines != 0, fld = ss->fld && lns;   // fld: the caller's key lines, step-major
    if (const int rc = check_key_line_fields(ctx, &frames, 1, !ss->fld, ss->fld && !lns, true)) return rc;
    const PlOrbDetectConfig* oc = &ss->oc;
    std::vector<int32_t> th0((size_t)2 * n);   // row 0 of the threshold table, [left n][right n]
    for (int k = 0; k < n; ++k) {
        if (fast_th0 && (fast_th0[k] < 0 || fast_th0[k] > 255)) return fail(ctx, PLSTVO_E_INVALID, "fast_th0 outside [0, 255]");
        th0[(size_t)k] = th0[(size_t)n + k] = fast_th0 && fast_th0[k] ? fast_th0[k] : oc->fast_threshold;
        if (th0[(size_t)k] < 0 || th0[(size_t)k] > 255)
            return fail(ctx, PLSTVO_E_INVALID, "ocfg->fast_threshold outside [0, 255] where fast_th0 leaves it");
    }
    if (T == 0) {   // nothing runs; row T of the thresholds is row 0
        if (fast_th) std::copy(th0.begin(), th0.begin() + n, fast_th);
        return 0;
    }
    if (n > 0 && (!ids || !results)) return fail(ctx, PLSTVO_E_INVALID, "null ids or results");
    if (2LL * n * T > 65535) return fail(ctx, PLSTVO_E_INVALID, "more than 65535 images in one call");
    if (const int rc = session_check_ids(ctx, ss, true, n, ids)) return rc;
    if (oc->n_features > PLSTVO_MAX_FEATURES)
        return fail(ctx, PLSTVO_E_INVALID, "ocfg.n_features exceeds PLSTVO_MAX_FEATURES: a step could fail on a feature limit");
    const PlCamera& cam = ss->cam;
    const bool pts = ss->cfg.has_points != 0;
    const int W = cam.width, H = cam.height, n_img = 2 * n * T;
    // the insert's checks (track_images_run) before any work: ORB's and LSD's plans, image sizes and pointers
    if (const int rc = orb_detect_check(ctx, oc)) return rc;
    if (pts && n > 0) {
        PlOrbConfig orb_cfg;
        OrbDevLevels levels;
        std::vector<int32_t> tabs;
        std::vector<size_t> tab_off;
        if (const int rc = orb_detect_levels(ctx, oc, W, H, orb_cfg, levels, tabs, tab_off)) return rc;
    }
    LsdLaunch lsd{};
    if (n > 0) {   // the session was created with an LSD config wherever it has lines
        if (const int rc = images_check(ctx, W, H, pts, lns, &frames, 1, lns && !fld ? &ss->lc : nullptr, n_img, lsd)) return rc;
    }
    // the key lines as line blocks: 2 t, 2 t + 1 are step t's left and right images (FLD: the caller's, cut here)
    const int nblk = 2 * T;
    LineBlocks lines;
    if (fld && n > 0)
        if (const int rc = lines.cut(ctx, &frames, 1, T, n)) return rc;
    if (n == 0) return 0;   // T empty inserts
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, ctx->img_ev.create());
    CK(ctx, ctx->img_join.create(cudaEventDisableTiming));
    ctx->img_timed = false;
    Events<2> run_ev;      // the call's start, the end of its uploads and preparation
    Events<3> marks[2];    // stereo step start, its end, tracking end, of even and odd steps
    CK(ctx, run_ev.create());
    CK(ctx, marks[0].create());
    CK(ctx, marks[1].create());
    cudaStream_t s = ctx->s_main;
    CK(ctx, cudaEventRecord(run_ev[0], s));
    const size_t px = (size_t)W * H, step_px = 2 * (size_t)n * px;
    const PlRectifier* rect = ss->rect;
    const bool prepare = rect && (pts || lns);
    // the threshold table [T + 1][2 n] (row t: step t's ORB thresholds, left and right), the results [T][n], and without a
    // rectifier the grey images, step-major: step t's n left images, then its n right images
    Arena a;
    const size_t o_img = a.take(prepare || !(pts || lns) ? 0 : (size_t)n_img * px), o_th = a.take((size_t)(T + 1) * 2 * n * 4),
                 o_res = a.take((size_t)T * n * sizeof(PlPoseResult));
    const bool keep = ss->retain;
    // the key-frame test: the streams' states [n], the decisions [T][n], and with retention each step's segments of the new
    // rows [T][n] (call order)
    size_t o_kfs = 0, o_kfr = 0, o_kfseg = 0;
    if (kc) {
        o_kfs = a.take((size_t)n * sizeof(PlKeyframeState));
        o_kfr = a.take((size_t)T * n * sizeof(PlKeyframeResult));
        o_kfseg = a.take(keep ? (size_t)T * n * sizeof(GatherSeg) : 0);
    }
    CK(ctx, a.alloc(ctx->arena_run));
    CK(ctx, a.up(o_th, th0.data(), th0.size() * 4, s));
    if (kc) CK(ctx, a.up(o_kfs, kf_state, (size_t)n * sizeof(PlKeyframeState), s));
    const double k_entropy = keyframe_k_entropy();
    std::vector<GatherSeg> kf_segs(kc && keep ? (size_t)T * n : 0);   // [T][n], as uploaded
    const int32_t* d_th = a.i32(o_th);
    const int ch = rect ? rect->channels : 1;
    std::vector<ImgPart> iparts;
    for (int t = 0; t < T; ++t) {
        iparts.push_back(ImgPart{frames->img_l + (size_t)t * n * px * ch, n});
        iparts.push_back(ImgPart{frames->img_r + (size_t)t * n * px * ch, n});
    }
    const uint8_t* d_img = nullptr;
    const uint8_t* d_rgb = nullptr;   // a colour FLD session's RGB2GRAY plane, which LBD reads
    SessionCall step = session_begin(ss, true, n, ids);   // step 0's; each later step's follows the commit of the one before
    if (prepare) {
        if (const int rc = rectify_call(ctx, rect, &step, n, n_img, iparts, s, &d_img, &d_rgb)) return rc;
    } else if (pts || lns) {
        size_t o = o_img;
        for (const ImgPart& ip : iparts) {
            CK(ctx, a.up(o, ip.p, (size_t)ip.n * px, s));
            o += (size_t)ip.n * px;
        }
        d_img = a.u8(o_img);
    }
    CK(ctx, cudaEventRecord(run_ev[1], s));
    // the lines of every image: LSD alone on the main stream (FLD: the caller's), then LBD on the second stream beside step
    // 0's ORB
    if (lns && !fld) {
        if (const int rc = lsd_enqueue(ctx, lsd, d_img, nullptr, {}, s)) return rc;
        if (const int rc = lines.take_lsd(ctx, &ss->lc, lsd, s, nblk, n)) return rc;
    }
    if (lines.run_lbd) {
        cudaEvent_t ready = next_event(ctx);
        CK(ctx, cudaEventRecord(ready, s));
        if (const int rc = lines.describe(ctx, W, H, d_rgb ? d_rgb : d_img, ready, {})) return rc;
    }
    float* ms = ctx->img_ms;
    std::fill(ms, ms + 5, 0.f);
    auto add_ms = [&](int k, cudaEvent_t from, cudaEvent_t to) -> int {
        float v = 0;
        CK(ctx, cudaEventElapsedTime(&v, from, to));
        ms[k] += v;
        return 0;
    };
    std::vector<int32_t> none((size_t)n + 1, 0), pl_off, pr_off;
    for (int t = 0; t < T; ++t) {
        if (t > 0) step = session_begin(ss, true, n, ids);
        step.retain = keep && (kc || t == T - 1);   // the retention arena holds the last step (every step for the key frames)
        OrbDetected orb;
        if (pts) {
            if (const int rc = orb_detect_enqueue(ctx, oc, 2 * n, W, H, d_img + (size_t)t * step_px, {}, nullptr, INT_MAX,
                                                  nullptr, orb, d_th + (size_t)t * 2 * n))
                return rc;
        } else {
            orb.off.assign((size_t)2 * n + 1, 0);
        }
        StereoSet sets[2];
        stereo_set_inputs(orb, 0, pts, lines, 2 * t, n, none, pl_off, pr_off, sets);
        StereoDevInputs dev;
        dev.lines_ready = lines.joined;
        cudaEvent_t* mk = marks[t % 2].ev;
        dev.marks = mk;
        dev.priors_resident = t > 0;   // step t - 1's handler update wrote them
        dev.tracked = [&](const Workspace& ws) -> int {
            CK(ctx, launch_session_handler(*h, n, ws.d_results.as<PlPoseResult>(), d_th + (size_t)t * 2 * n,
                                           a.i32(o_th) + (size_t)(t + 1) * 2 * n, ws.d_priors.as<PlPrior>(),
                                           a.at<PlPoseResult>(o_res) + (size_t)t * n, s));
            ctx->launches++;
            if (kc) {
                PlKeyframeResult* d_kf = a.at<PlKeyframeResult>(o_kfr) + (size_t)t * n;
                CK(ctx, launch_session_keyframe(*kc, k_entropy, n, ws.d_results.as<PlPoseResult>(), a.at<PlKeyframeState>(o_kfs),
                                                d_kf, ws.d_priors.as<PlPrior>(), s));
                ctx->launches++;
                if (keep) {   // the key frames' rows, from this step's retention arena into its own chunk, at the same rows
                    GatherSeg* seg = kf_segs.data() + (size_t)t * n;
                    int32_t np = 0, nl = 0;
                    for (int k = 0; k < n; ++k) {
                        seg[k] = GatherSeg{np, np, step.new_pt[(size_t)k], nl, nl, step.new_ls[(size_t)k]};
                        np += seg[k].n_pt;
                        nl += seg[k].n_ls;
                    }
                    const size_t o = o_kfseg + (size_t)t * n * sizeof(GatherSeg);
                    CK(ctx, a.up(o, seg, (size_t)n * sizeof(GatherSeg), s));
                    ss->kf_steps.push_back(std::unique_ptr<SessionRetained>(new SessionRetained()));
                    SessionRetained& c = *ss->kf_steps.back();
                    CK(ctx, c.lay_out((size_t)np, (size_t)nl, 0, 0));
                    CK(ctx, launch_session_gather(ss->kept.rec, c.rec, false, a.at<GatherSeg>(o), n, s, d_kf));
                    ctx->launches++;
                }
            }
            CK(ctx, cudaEventRecord(mk[2], s));
            // An insert ends synchronised; a step does not, and the next step's stereo step and tracker plan upload into the
            // same arenas on s_h2d (offsets, line angles, problem tables) while this step's lifts and solver may still read
            // them on s_main.  Every later upload on s_h2d waits for this step's end.
            cudaEvent_t step_done = next_event(ctx);
            CK(ctx, cudaEventRecord(step_done, s));
            CK(ctx, cudaStreamWaitEvent(ctx->s_h2d, step_done, 0));
            return 0;
        };
        int32_t* ns = n_stereo ? n_stereo + (size_t)t * 4 * n : nullptr;
        const int rc = track_stereo_common(ctx, &cam, &ss->cfg, &ss->mc, &ss->sc, sets, nullptr, t == 0 ? priors : nullptr,
                                           results + (size_t)t * n, ns, false, -1, &dev, &step);
        if (rc) return rc;
        session_commit(step);
        // the stereo step's count readback synchronised the main stream: this step's ORB and the last step are done
        if (pts)
            if (const int rc2 = add_ms(1, ctx->orb_det_ev[0], ctx->orb_det_ev[4])) return rc2;
        if (t > 0) {
            const cudaEvent_t* pm = marks[(t - 1) % 2].ev;
            if (const int rc2 = add_ms(3, pm[0], pm[1])) return rc2;
            if (const int rc2 = add_ms(4, pm[1], pm[2])) return rc2;
        }
    }
    CK(ctx, a.down(results, o_res, (size_t)T * n * sizeof(PlPoseResult), s));
    std::vector<PlKeyframeState> kfs_out(kc ? (size_t)n : 0);
    if (kc) {
        CK(ctx, a.down(kf, o_kfr, (size_t)T * n * sizeof(PlKeyframeResult), s));
        CK(ctx, a.down(kfs_out.data(), o_kfs, (size_t)n * sizeof(PlKeyframeState), s));
    }
    if (fast_th)
        CK(ctx, cudaMemcpy2DAsync(fast_th, (size_t)n * 4, d_th, (size_t)2 * n * 4, (size_t)n * 4, (size_t)T + 1,
                                  cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    CK(ctx, cudaStreamSynchronize(ctx->s_alt));
    const cudaEvent_t* pm = marks[(T - 1) % 2].ev;
    if (const int rc = add_ms(3, pm[0], pm[1])) return rc;
    if (const int rc = add_ms(4, pm[1], pm[2])) return rc;
    if (const int rc = add_ms(0, run_ev[0], run_ev[1])) return rc;
    if (lns && !fld)
        if (const int rc = add_ms(2, ctx->lsd_ev[0], lines.run_lbd ? ctx->lbd_ev[2] : ctx->lsd_ev[5])) return rc;
    if (fld && lines.run_lbd)
        if (const int rc = add_ms(2, ctx->lbd_ev[0], ctx->lbd_ev[2])) return rc;
    ctx->img_timed = true;
    if (kc) {
        std::copy(kfs_out.begin(), kfs_out.end(), kf_state);
        for (int t = 0; keep && t < T; ++t)
            for (int k = 0; k < n; ++k) {
                if (!kf[(size_t)t * n + k].new_kf) continue;
                const GatherSeg& g = kf_segs[(size_t)t * n + k];
                ss->kf_rows.insert(ss->kf_rows.end(), {t, ids[k], g.n_pt, g.n_ls});
                ss->kf_off.insert(ss->kf_off.end(), {g.src_pt, g.src_ls});
            }
    }
    return 0;
}

// One group of a scheduled run: a step's initialize entries or its insert entries, which the chain hands to one session call
struct SchedGroup {
    int t = 0;
    bool track = false;
    std::vector<int32_t> ids;   // the group's streams, in the order of the call's ids
    std::vector<int> pos;       // their call positions: their state slots
    std::vector<int> frame;     // their frames' indices in frames
    int img0 = 0;               // the group's first image on the device: its left images, then its right ones
    int e0 = 0, r0 = 0;         // its first entry in the entry table, and (insert) its first row of the insert results
};

// plstvo_stereo_session_run_schedule after the context lock: the checks, then each step's initialize group and insert group
// as the chain's two calls.  The present images go up, are prepared and have their key lines found and described once, in
// group order; each stream's FAST threshold, prior and key-frame state live in a device slot for the whole call, gathered
// for an insert group's ORB, solver and test by session_schedule_gather_kernel and written back (reset after an initialize)
// by session_schedule_update_kernel.  *ran: some group ran; *last_track, *last_n: the last group (what retention holds).
int session_schedule(PlContext* ctx, PlStereoSession* ss, const PlHandlerConfig* h, const PlKeyframeConfig* kc, int n,
                     const int32_t* ids, int T, const uint8_t* schedule, const PlStereoImages* frames, const int32_t* fast_th0,
                     const PlPrior* priors, PlKeyframeState* kf_state, PlPoseResult* results, PlKeyframeResult* kf,
                     int32_t* fast_th, int32_t* n_stereo, bool* ran, bool* last_track, int* last_n) {
    if (const int rc = handler_check(ctx, h)) return rc;
    if (T < 0) return fail(ctx, PLSTVO_E_INVALID, "negative T");
    if (n < 0 || !frames) return fail(ctx, PLSTVO_E_INVALID, "null frames or negative n");
    const long long TN = (long long)T * n;
    if (TN > 0 && !schedule) return fail(ctx, PLSTVO_E_INVALID, "null schedule");
    long long B = 0;
    for (long long i = 0; i < TN; ++i) {
        if (schedule[i] > 2) return fail(ctx, PLSTVO_E_INVALID, "schedule value outside {0, 1, 2}");
        B += schedule[i] != 0;
    }
    if ((long long)frames->B != B) return fail(ctx, PLSTVO_E_SIZE, "frames->B differs from the schedule's non-zero entries");
    const bool lns = ss->cfg.has_lines != 0, fld = ss->fld && lns;   // fld: the caller's key lines, in frames' order
    if (const int rc = check_key_line_fields(ctx, &frames, 1, !ss->fld, ss->fld && !lns, false)) return rc;
    const PlOrbDetectConfig* oc = &ss->oc;
    std::vector<int32_t> th0((size_t)n);
    for (int k = 0; k < n; ++k) {
        if (fast_th0 && (fast_th0[k] < 0 || fast_th0[k] > 255)) return fail(ctx, PLSTVO_E_INVALID, "fast_th0 outside [0, 255]");
        th0[(size_t)k] = fast_th0 && fast_th0[k] ? fast_th0[k] : oc->fast_threshold;
        if (th0[(size_t)k] < 0 || th0[(size_t)k] > 255)
            return fail(ctx, PLSTVO_E_INVALID, "ocfg->fast_threshold outside [0, 255] where fast_th0 leaves it");
    }
    auto all_rows = [&]() {   // no group runs: every threshold row is row 0
        for (int t = 0; fast_th && t <= T; ++t) std::copy(th0.begin(), th0.end(), fast_th + (size_t)t * n);
    };
    if (T == 0) {
        all_rows();
        return 0;
    }
    if (n > 0 && (!ids || !results)) return fail(ctx, PLSTVO_E_INVALID, "null ids or results");
    if (2 * B > 65535) return fail(ctx, PLSTVO_E_INVALID, "more than 65535 images in one call");
    if (const int rc = session_check_ids(ctx, ss, false, n, ids)) return rc;
    // which stream holds a frame at each entry (held at the call's start, or initialised at an earlier step of it), and the
    // initialize entries' thresholds
    std::vector<uint8_t> live((size_t)n);
    for (int k = 0; k < n; ++k) live[(size_t)k] = ss->live[(size_t)ids[k]];
    std::vector<int32_t> entry_th((size_t)B, 0), frame_of((size_t)TN, -1);
    for (long long i = 0, b = 0; i < TN; ++i) {
        const int code = schedule[i], k = (int)(i % n);
        if (!code) continue;
        const int32_t ft = frames->fast_th ? frames->fast_th[b] : 0;
        if (code == 1 && !live[(size_t)k])
            return fail(ctx, PLSTVO_E_INVALID, "insert on a stream with no frame at that step: initialize it first, before or in the call");
        if (code == 1 && ft) return fail(ctx, PLSTVO_E_INVALID, "frames->fast_th of an insert entry must be 0: the run sets its thresholds");
        if (code == 2) {
            entry_th[(size_t)b] = ft ? ft : oc->fast_threshold;
            if (entry_th[(size_t)b] < 0 || entry_th[(size_t)b] > 255)
                return fail(ctx, PLSTVO_E_INVALID, "an initialize entry's threshold outside [0, 255]");
            live[(size_t)k] = 1;
        }
        frame_of[(size_t)i] = (int32_t)b++;
    }
    if (oc->n_features > PLSTVO_MAX_FEATURES)
        return fail(ctx, PLSTVO_E_INVALID, "ocfg.n_features exceeds PLSTVO_MAX_FEATURES: a step could fail on a feature limit");
    const PlCamera& cam = ss->cam;
    const bool pts = ss->cfg.has_points != 0;
    const int W = cam.width, H = cam.height, n_img = (int)(2 * B);
    if (const int rc = orb_detect_check(ctx, oc)) return rc;
    if (pts && B > 0) {
        PlOrbConfig orb_cfg;
        OrbDevLevels levels;
        std::vector<int32_t> tabs;
        std::vector<size_t> tab_off;
        if (const int rc = orb_detect_levels(ctx, oc, W, H, orb_cfg, levels, tabs, tab_off)) return rc;
    }
    LsdLaunch lsd{};
    if (B > 0)
        if (const int rc = images_check(ctx, W, H, pts, lns, &frames, 1, lns && !fld ? &ss->lc : nullptr, n_img, lsd)) return rc;
    // the groups in chain order, the entry table, and the device order of the images (frame, side)
    std::vector<SchedGroup> groups;
    std::vector<SchedEntry> entries;
    std::vector<int> img_frame, img_side;
    int n_ins = 0, max_e = 0, max_ins = 0;
    for (int t = 0; t < T; ++t)
        for (int code : {2, 1}) {
            SchedGroup g;
            g.t = t;
            g.track = code == 1;
            for (int k = 0; k < n; ++k)
                if (schedule[(size_t)t * n + k] == code) {
                    g.ids.push_back(ids[k]);
                    g.pos.push_back(k);
                    g.frame.push_back(frame_of[(size_t)t * n + k]);
                }
            const int ne = (int)g.ids.size();
            if (!ne) continue;
            g.img0 = (int)img_frame.size();
            g.e0 = (int)entries.size();
            g.r0 = n_ins;
            for (int i = 0; i < ne; ++i) entries.push_back(SchedEntry{g.pos[(size_t)i], entry_th[(size_t)g.frame[(size_t)i]]});
            for (int side = 0; side < 2; ++side)
                for (int i = 0; i < ne; ++i) {
                    img_frame.push_back(g.frame[(size_t)i]);
                    img_side.push_back(side);
                }
            if (g.track) {
                n_ins += ne;
                max_ins = std::max(max_ins, ne);
            }
            max_e = std::max(max_e, ne);
            groups.push_back(std::move(g));
        }
    LineBlocks lines;   // one block per device image
    if (fld && B > 0)
        if (const int rc = lines.cut_images(ctx, frames, img_frame, img_side)) return rc;
    if (B == 0) {   // every stream idles at every step
        all_rows();
        return 0;
    }
    *ran = true;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, ctx->img_ev.create());
    CK(ctx, ctx->img_join.create(cudaEventDisableTiming));
    ctx->img_timed = false;
    Events<2> run_ev;      // the call's start, the end of its uploads and preparation
    Events<3> marks[2];    // stereo step start, its end, tracking end, of even and odd groups
    CK(ctx, run_ev.create());
    CK(ctx, marks[0].create());
    CK(ctx, marks[1].create());
    cudaStream_t s = ctx->s_main;
    CK(ctx, cudaEventRecord(run_ev[0], s));
    const size_t px = (size_t)W * H;
    const PlRectifier* rect = ss->rect;
    const bool prepare = rect && (pts || lns);
    const bool rgb = prepare && ss->fld && lns && rect->channels > 1;   // rectify_call's RGB2GRAY plane, which LBD reads
    const bool keep = ss->retain;
    // the grey images in group order; the entry table; the slots (thresholds [n], priors [n], key-frame states [n]); the
    // slots' thresholds before each step with entries and after the last ([T + 1][n]); an insert group's ORB threshold row
    // and the handler's next row ([2 max_ins] each); the insert results [n_ins], and with the test the group's states, the
    // decisions [n_ins] and with retention the key frames' segments [n_ins]
    Arena a;
    const size_t o_img = a.take(pts || lns ? (size_t)n_img * px : 0), o_rgb = a.take(rgb ? (size_t)n_img * px : 0),
                 o_ent = a.take(entries.size() * sizeof(SchedEntry)), o_ths = a.take((size_t)n * 4),
                 o_pri = a.take((size_t)n * sizeof(PlPrior)), o_snap = a.take((size_t)(T + 1) * n * 4),
                 o_th = a.take((size_t)2 * max_ins * 4), o_thn = a.take((size_t)2 * max_ins * 4),
                 o_res = a.take((size_t)n_ins * sizeof(PlPoseResult));
    size_t o_kfs = 0, o_kfst = 0, o_kfr = 0, o_kfseg = 0;
    if (kc) {
        o_kfs = a.take((size_t)n * sizeof(PlKeyframeState));
        o_kfst = a.take((size_t)max_ins * sizeof(PlKeyframeState));
        o_kfr = a.take((size_t)n_ins * sizeof(PlKeyframeResult));
        o_kfseg = a.take(keep ? (size_t)n_ins * sizeof(GatherSeg) : 0);
    }
    CK(ctx, a.alloc(ctx->arena_run));
    // the insert groups' priors are gathered straight into the workspace's, which no group then regrows
    CK(ctx, ctx->ws.d_priors.ensure((size_t)std::max(max_ins, 1) * sizeof(PlPrior)));
    PlPrior fresh{};   // priorOf of a freshly initialised frame; priors NULL starts every stream from it
    for (int i = 0; i < 16; ++i) fresh.Tfw[i] = fresh.DT[i] = (i % 5 == 0) ? 1.0 : 0.0;
    for (int i = 0; i < 36; ++i) fresh.Tfw_cov[i] = (i % 7 == 0) ? 1.0 : 0.0;
    fresh.err_norm = -1.0;
    const std::vector<PlPrior> pri0 = priors ? std::vector<PlPrior>(priors, priors + n) : std::vector<PlPrior>((size_t)n, fresh);
    CK(ctx, a.up(o_ent, entries.data(), entries.size() * sizeof(SchedEntry), s));
    CK(ctx, a.up(o_ths, th0.data(), (size_t)n * 4, s));
    CK(ctx, a.up(o_pri, pri0.data(), (size_t)n * sizeof(PlPrior), s));
    if (kc) CK(ctx, a.up(o_kfs, kf_state, (size_t)n * sizeof(PlKeyframeState), s));
    const SchedEntry* d_ent = a.at<SchedEntry>(o_ent);
    int32_t* d_ths = a.at<int32_t>(o_ths);
    PlPrior* d_pri = a.at<PlPrior>(o_pri);
    PlKeyframeState* d_kfs = kc ? a.at<PlKeyframeState>(o_kfs) : nullptr;
    int32_t* d_th = a.at<int32_t>(o_th);
    int32_t* d_thn = a.at<int32_t>(o_thn);
    uint8_t* d_img = a.u8(o_img);
    const uint8_t* d_rgb = rgb ? a.u8(o_rgb) : nullptr;
    const int ch = rect ? rect->channels : 1;
    auto host_image = [&](int z) {
        return (img_side[(size_t)z] ? frames->img_r : frames->img_l) + (size_t)img_frame[(size_t)z] * px * ch;
    };
    if (prepare) {   // per group, as its streams' rectifiers take them; the prepared images are copied into group order
        for (const SchedGroup& g : groups) {
            const int ne = (int)g.ids.size();
            std::vector<ImgPart> parts;
            for (int z = g.img0; z < g.img0 + 2 * ne; ++z) parts.push_back(ImgPart{host_image(z), 1});
            const SessionCall gc{ss, g.track, false, ne, g.ids.data()};
            const uint8_t* out = nullptr;
            const uint8_t* out_rgb = nullptr;
            if (const int rc = rectify_call(ctx, rect, &gc, ne, 2 * ne, parts, s, &out, &out_rgb)) return rc;
            CK(ctx, cudaMemcpyAsync(d_img + (size_t)g.img0 * px, out, 2 * ne * px, cudaMemcpyDeviceToDevice, s));
            if (rgb)
                CK(ctx, cudaMemcpyAsync(a.u8(o_rgb) + (size_t)g.img0 * px, out_rgb, 2 * ne * px, cudaMemcpyDeviceToDevice, s));
        }
    } else if (pts || lns) {   // runs of consecutive host images in one copy each
        for (int z = 0; z < n_img;) {
            int e = z + 1;
            while (e < n_img && host_image(e) == host_image(e - 1) + px) ++e;
            CK(ctx, a.up(o_img + (size_t)z * px, host_image(z), (size_t)(e - z) * px, s));
            z = e;
        }
    }
    CK(ctx, cudaEventRecord(run_ev[1], s));
    // the lines of every image: LSD alone on the main stream (FLD: the caller's), then LBD on the second stream beside the
    // first group's ORB
    if (lns && !fld) {
        if (const int rc = lsd_enqueue(ctx, lsd, d_img, nullptr, {}, s)) return rc;
        if (const int rc = lines.take_lsd(ctx, &ss->lc, lsd, s, n_img, 1)) return rc;
    }
    if (lines.run_lbd) {
        cudaEvent_t ready = next_event(ctx);
        CK(ctx, cudaEventRecord(ready, s));
        if (const int rc = lines.describe(ctx, W, H, d_rgb ? d_rgb : d_img, ready, {})) return rc;
    }
    float* ms = ctx->img_ms;
    std::fill(ms, ms + 5, 0.f);
    auto add_ms = [&](int k, cudaEvent_t from, cudaEvent_t to) -> int {
        float v = 0;
        CK(ctx, cudaEventElapsedTime(&v, from, to));
        ms[k] += v;
        return 0;
    };
    const double k_entropy = keyframe_k_entropy();
    std::vector<GatherSeg> kf_segs(kc && keep ? (size_t)n_ins : 0);   // [n_ins], as uploaded
    const LineBlocks no_lines;
    std::vector<int32_t> none((size_t)max_e + 1, 0), pl_off, pr_off, l_off, r_off, ns((size_t)4 * max_e);
    std::vector<float> ang;
    std::vector<int32_t> th_init;
    int last_t = -1;
    for (size_t j = 0; j < groups.size(); ++j) {
        const SchedGroup& g = groups[j];
        const int ne = (int)g.ids.size();
        if (g.t != last_t) {   // the slots' thresholds before the step
            CK(ctx, cudaMemcpyAsync(a.u8(o_snap) + (size_t)g.t * n * 4, d_ths, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
            last_t = g.t;
        }
        SessionCall step = session_begin(ss, g.track, ne, g.ids.data());
        // the retention arena holds the last group (every insert group's rows for the key frames)
        step.retain = keep && (j + 1 == groups.size() || (kc && g.track));
        if (g.track) {
            CK(ctx, launch_session_schedule_gather(ne, d_ent + g.e0, d_ths, d_pri, d_kfs, d_th, ctx->ws.d_priors.as<PlPrior>(),
                                                   kc ? a.at<PlKeyframeState>(o_kfst) : nullptr, s));
            ctx->launches++;
        } else {   // initialize: each frame at its entry's threshold, from the host as _initialize takes it
            th_init.assign((size_t)2 * ne, 0);
            for (int i = 0; i < ne; ++i) th_init[(size_t)i] = th_init[(size_t)(ne + i)] = entries[(size_t)(g.e0 + i)].th;
        }
        OrbDetected orb;
        if (pts) {
            if (const int rc = orb_detect_enqueue(ctx, oc, 2 * ne, W, H, d_img + (size_t)g.img0 * px, {},
                                                  g.track ? nullptr : th_init.data(), INT_MAX, nullptr, orb,
                                                  g.track ? d_th : nullptr))
                return rc;
        } else {
            orb.off.assign((size_t)2 * ne + 1, 0);
        }
        StereoSet sets[2];
        stereo_set_inputs(orb, 0, pts, no_lines, 0, ne, none, pl_off, pr_off, sets);
        schedule_line_inputs(lines, g.img0, ne, l_off, r_off, ang, sets[1]);
        StereoDevInputs dev;
        dev.lines_ready = lines.joined;
        cudaEvent_t* mk = marks[j % 2].ev;
        dev.marks = mk;
        if (g.track) {
            dev.priors_resident = true;   // gathered above
            dev.tracked = [&](const Workspace& ws) -> int {
                PlPrior* wp = ws.d_priors.as<PlPrior>();
                PlKeyframeState* kfst = kc ? a.at<PlKeyframeState>(o_kfst) : nullptr;
                CK(ctx, launch_session_handler(*h, ne, ws.d_results.as<PlPoseResult>(), d_th, d_thn, wp,
                                               a.at<PlPoseResult>(o_res) + g.r0, s));
                ctx->launches++;
                if (kc) {
                    PlKeyframeResult* d_kf = a.at<PlKeyframeResult>(o_kfr) + g.r0;
                    CK(ctx, launch_session_keyframe(*kc, k_entropy, ne, ws.d_results.as<PlPoseResult>(), kfst, d_kf, wp, s));
                    ctx->launches++;
                    if (keep) {   // as session_run: the key frames' rows into the step's own chunk (chunk t: step t)
                        GatherSeg* seg = kf_segs.data() + g.r0;
                        int32_t np = 0, nl = 0;
                        for (int i = 0; i < ne; ++i) {
                            seg[i] = GatherSeg{np, np, step.new_pt[(size_t)i], nl, nl, step.new_ls[(size_t)i]};
                            np += seg[i].n_pt;
                            nl += seg[i].n_ls;
                        }
                        const size_t o = o_kfseg + (size_t)g.r0 * sizeof(GatherSeg);
                        CK(ctx, a.up(o, seg, (size_t)ne * sizeof(GatherSeg), s));
                        while (ss->kf_steps.size() < (size_t)g.t)   // steps without inserts keep an empty chunk
                            ss->kf_steps.push_back(std::unique_ptr<SessionRetained>(new SessionRetained()));
                        ss->kf_steps.push_back(std::unique_ptr<SessionRetained>(new SessionRetained()));
                        SessionRetained& c = *ss->kf_steps.back();
                        CK(ctx, c.lay_out((size_t)np, (size_t)nl, 0, 0));
                        CK(ctx, launch_session_gather(ss->kept.rec, c.rec, false, a.at<GatherSeg>(o), ne, s, d_kf));
                        ctx->launches++;
                    }
                }
                CK(ctx, launch_session_schedule_update(ne, d_ent + g.e0, false, d_thn, wp, kfst, d_ths, d_pri, d_kfs, s));
                ctx->launches++;
                CK(ctx, cudaEventRecord(mk[2], s));
                // as session_run: later uploads on s_h2d wait for this group's end
                cudaEvent_t step_done = next_event(ctx);
                CK(ctx, cudaEventRecord(step_done, s));
                CK(ctx, cudaStreamWaitEvent(ctx->s_h2d, step_done, 0));
                return 0;
            };
        }
        const int rc = track_stereo_common(ctx, &cam, &ss->cfg, &ss->mc, &ss->sc, sets, nullptr, nullptr, results,
                                           n_stereo ? ns.data() : nullptr, false, -1, &dev, &step);
        if (rc) return rc;
        if (!g.track) {
            CK(ctx, launch_session_schedule_update(ne, d_ent + g.e0, true, nullptr, nullptr, nullptr, d_ths, d_pri, d_kfs, s));
            ctx->launches++;
        }
        session_commit(step);
        for (int i = 0; n_stereo && i < ne; ++i) {   // an initialize entry's row: {0, 0, points, lines}
            int32_t* row = n_stereo + ((size_t)g.t * n + g.pos[(size_t)i]) * 4;
            for (int c = 0; c < 4; ++c)
                row[c] = g.track ? ns[(size_t)4 * i + c] : c < 2 ? 0 : ns[(size_t)2 * i + c - 2];
        }
        // the stereo step's count readback synchronised the main stream: this group's ORB and the last group are done
        if (pts)
            if (const int rc2 = add_ms(1, ctx->orb_det_ev[0], ctx->orb_det_ev[4])) return rc2;
        if (j > 0) {
            const cudaEvent_t* pm = marks[(j - 1) % 2].ev;
            if (const int rc2 = add_ms(3, pm[0], pm[1])) return rc2;
            if (const int rc2 = add_ms(4, pm[1], pm[2])) return rc2;
        }
    }
    CK(ctx, cudaMemcpyAsync(a.u8(o_snap) + (size_t)T * n * 4, d_ths, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    std::vector<PlPoseResult> res((size_t)n_ins);
    std::vector<PlKeyframeResult> kres(kc ? (size_t)n_ins : 0);
    std::vector<PlKeyframeState> kfs_out(kc ? (size_t)n : 0);
    std::vector<int32_t> snap((size_t)(T + 1) * n);
    CK(ctx, a.down(res.data(), o_res, res.size() * sizeof(PlPoseResult), s));
    if (kc) {
        CK(ctx, a.down(kres.data(), o_kfr, kres.size() * sizeof(PlKeyframeResult), s));
        CK(ctx, a.down(kfs_out.data(), o_kfs, (size_t)n * sizeof(PlKeyframeState), s));
    }
    CK(ctx, a.down(snap.data(), o_snap, snap.size() * 4, s));
    CK(ctx, cudaStreamSynchronize(s));
    CK(ctx, cudaStreamSynchronize(ctx->s_alt));
    const cudaEvent_t* pm = marks[(groups.size() - 1) % 2].ev;
    if (const int rc = add_ms(3, pm[0], pm[1])) return rc;
    if (const int rc = add_ms(4, pm[1], pm[2])) return rc;
    if (const int rc = add_ms(0, run_ev[0], run_ev[1])) return rc;
    if (lns && !fld)
        if (const int rc = add_ms(2, ctx->lsd_ev[0], lines.run_lbd ? ctx->lbd_ev[2] : ctx->lsd_ev[5])) return rc;
    if (fld && lines.run_lbd)
        if (const int rc = add_ms(2, ctx->lbd_ev[0], ctx->lbd_ev[2])) return rc;
    ctx->img_timed = true;
    // the insert entries' rows; the threshold rows: row t is the slots before the next step with entries (or after the last
    // step), with each initialize entry's threshold in place
    std::vector<uint8_t> has_entries((size_t)T, 0);
    for (const SchedGroup& g : groups) {
        has_entries[(size_t)g.t] = 1;
        for (int i = 0; g.track && i < (int)g.ids.size(); ++i) {
            const size_t at = (size_t)g.t * n + g.pos[(size_t)i], r = (size_t)(g.r0 + i);
            results[at] = res[r];
            if (kc) kf[at] = kres[r];
        }
    }
    if (fast_th) {
        for (int t = T, next = T; t >= 0; --t) {
            if (t < T && has_entries[(size_t)t]) next = t;
            std::copy(snap.begin() + (size_t)next * n, snap.begin() + (size_t)(next + 1) * n, fast_th + (size_t)t * n);
        }
        for (const SchedGroup& g : groups)
            for (int i = 0; !g.track && i < (int)g.ids.size(); ++i)
                fast_th[(size_t)g.t * n + g.pos[(size_t)i]] = entries[(size_t)(g.e0 + i)].th;
    }
    if (kc) {
        std::copy(kfs_out.begin(), kfs_out.end(), kf_state);
        for (const SchedGroup& g : groups)
            for (int i = 0; keep && g.track && i < (int)g.ids.size(); ++i) {
                const size_t r = (size_t)(g.r0 + i);
                if (!kres[r].new_kf) continue;
                const GatherSeg& sg = kf_segs[r];
                ss->kf_rows.insert(ss->kf_rows.end(), {g.t, g.ids[(size_t)i], sg.n_pt, sg.n_ls});
                ss->kf_off.insert(ss->kf_off.end(), {sg.src_pt, sg.src_ls});
            }
    }
    *last_track = groups.back().track;
    *last_n = (int)groups.back().ids.size();
    return 0;
}
}  // namespace

int plstvo_stereo_session_run(PlContext* ctx, PlStereoSession* ss, const PlHandlerConfig* h, int n, const int32_t* ids, int T,
                              const PlStereoImages* frames, const int32_t* fast_th0, const PlPrior* priors,
                              PlPoseResult* results, int32_t* fast_th, int32_t* n_stereo) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, ss)) return rc;
    session_start(ss, false);   // a run of T = 0 leaves what the last call retained readable
    const int rc = session_run(ctx, ss, h, n, ids, T, frames, fast_th0, priors, results, fast_th, n_stereo);
    return session_finish(ctx, ss, rc, true, n, T > 0);
}

/* ---- the same loop with the key-frame test ---- */
void plstvo_default_keyframe_config(PlKeyframeConfig* k) {
    if (!k) return;
    k->min_entropy_ratio = 0.85; k->max_kf_t_dist = 5.0; k->max_kf_r_dist = 15.0;
}

void plstvo_initial_keyframe_state(PlKeyframeState* s) {
    if (!s) return;
    memset(s, 0, sizeof *s);
    s->prev_f_iskf = 1;
    for (int i = 0; i < 4; ++i) s->T_prevKF[5 * i] = 1.0;
}

int plstvo_stereo_session_run_keyframes(PlContext* ctx, PlStereoSession* ss, const PlHandlerConfig* h, const PlKeyframeConfig* k,
                                        int n, const int32_t* ids, int T, const PlStereoImages* frames, const int32_t* fast_th0,
                                        const PlPrior* priors, PlKeyframeState* kf_state, PlPoseResult* results,
                                        PlKeyframeResult* kf, int32_t* fast_th, int32_t* n_stereo) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, ss)) return rc;
    session_start(ss, true);   // what the last call retained is discarded, also by a run of T = 0
    if (const int rc = keyframe_check(ctx, k, n, kf_state, kf)) return rc;
    const int rc = session_run(ctx, ss, h, n, ids, T, frames, fast_th0, priors, results, fast_th, n_stereo, k, kf_state, kf);
    if (session_finish(ctx, ss, rc, true, n, T > 0) == 0) ss->kf_valid = ss->retain;
    return rc;
}

int plstvo_stereo_session_run_schedule(PlContext* ctx, PlStereoSession* ss, const PlHandlerConfig* h, const PlKeyframeConfig* k,
                                       int n, const int32_t* ids, int T, const uint8_t* schedule, const PlStereoImages* frames,
                                       const int32_t* fast_th0, const PlPrior* priors, PlKeyframeState* kf_state,
                                       PlPoseResult* results, PlKeyframeResult* kf, int32_t* fast_th, int32_t* n_stereo) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, ss)) return rc;
    session_start(ss, k != nullptr);   // as _run (k NULL) or _run_keyframes leaves what the last call retained
    if (k) {
        if (const int rc = keyframe_check(ctx, k, n, kf_state, kf)) return rc;
    } else if (kf_state || kf) {
        return fail(ctx, PLSTVO_E_INVALID, "kf_state and kf must be NULL without a key-frame config");
    }
    bool ran = false, track = false;
    int last_n = 0;
    const int rc = session_schedule(ctx, ss, h, k, n, ids, T, schedule, frames, fast_th0, priors, kf_state, results, kf, fast_th,
                                    n_stereo, &ran, &track, &last_n);
    if (session_finish(ctx, ss, rc, track, last_n, ran) == 0 && k) ss->kf_valid = ss->retain;
    return rc;
}

int plstvo_stereo_session_read_keyframes(PlContext* ctx, const PlStereoSession* ss, const PlStereoFrameOut* out, int32_t* rows) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (const int rc = session_check(ctx, out ? ss : nullptr, "null session or output")) return rc;
    if (!ss->retain) return fail(ctx, PLSTVO_E_INVALID, "retention is off: plstvo_stereo_session_retain(ctx, s, 1) first");
    if (!ss->kf_valid) return fail(ctx, PLSTVO_E_INVALID, "no key frames kept: the last call on the session was not a successful run_keyframes");
    CK(ctx, cudaSetDevice(ctx->device));
    const RecPtrs dst = frame_out_records(out);
    const int n_kf = (int)(ss->kf_rows.size() / 4);
    cudaStream_t s = ctx->s_main;
    size_t at_pt = 0, at_ls = 0;   // rows copied so far
    for (int j = 0; j < n_kf; ++j) {
        const int32_t* r = ss->kf_rows.data() + 4 * (size_t)j;
        const SessionRetained& c = *ss->kf_steps[(size_t)r[0]];
        for (int a = 0; a < N_LIFT; ++a) {
            const bool pt = rec_is_point(a);
            const size_t w = (size_t)REC_BYTES[a], rows_j = (size_t)(pt ? r[2] : r[3]);
            const size_t from = (size_t)ss->kf_off[2 * (size_t)j + (pt ? 0 : 1)], to = pt ? at_pt : at_ls;
            if (dst.p[a] && rows_j)
                CK(ctx, cudaMemcpyAsync(dst.at<uint8_t>(a) + to * w, c.rec.at<uint8_t>(a) + from * w, rows_j * w,
                                        cudaMemcpyDeviceToHost, s));
        }
        at_pt += (size_t)r[2];
        at_ls += (size_t)r[3];
    }
    CK(ctx, cudaStreamSynchronize(s));
    if (rows) std::copy(ss->kf_rows.begin(), ss->kf_rows.end(), rows);
    return n_kf;
}

int plstvo_track_stereo_images_stage_times(PlContext* ctx, float ms5[5]) {
    if (!ctx || !ms5) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!ctx->img_timed) return fail(ctx, PLSTVO_E_INVALID, "no images call on this context yet");
    memcpy(ms5, ctx->img_ms, sizeof(ctx->img_ms));
    return 0;
}

}  // extern "C"
