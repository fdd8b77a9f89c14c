// plstvo.hpp — header-only C++17 host layer over the C-ABI (plstvo.h): RAII context plus a StereoFrameHandler with
// the reference's method names (include/stereoFrameHandler.h:41-54) for frames of pre-extracted features, a
// StereoImageHandler with the same names for stereo images alone, and a StereoStreamsHandler that runs one such handler per
// camera over a StereoSession (each stream's previous frame kept on the device).  It has no
// Eigen / OpenCV dependency; the Eigen/OpenCV shim that makes it a drop-in for libstvo.so is in INTEGRATION.md.
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "plstvo.h"

namespace plstvo {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

class Context {
public:
    explicit Context(int device = -1) {
        const int rc = plstvo_create(device, &ctx_);
        if (rc != 0) throw Error(rc, "plstvo_create failed: no sm_90 CUDA device (there is no CPU fallback)");
    }
    ~Context() { plstvo_destroy(ctx_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    PlContext* get() const { return ctx_; }
    int check(int rc) const {   // the reference throws std::runtime_error where the C-ABI returns a negative code
        if (rc < 0) throw Error(rc, plstvo_last_error(ctx_));
        return rc;
    }
private:
    PlContext* ctx_ = nullptr;
};

// One stereo frame's pre-extracted features (StereoFrame::stereo_pt / stereo_ls / pdesc_l / ldesc_l), SoA.
struct StereoFrame {
    std::vector<uint8_t> pdesc, ldesc;                                   // [n][32], [m][32]
    std::vector<double> pt_P, pt_pl, pt_sigma2;                          // [n][3], [n][2], [n]
    std::vector<double> ls_sP, ls_eP, ls_le, ls_spl, ls_epl, ls_sigma2;  // [m][3] x3, [m][2] x2, [m]
    std::vector<int32_t> ls_level;                                       // [m]
    // the rest of stereo_pt / stereo_ls, filled by the images handlers' keepFeatures (the tracker does not read them):
    // disparities, ORB octave, start / end disparities, line angle, and each feature's index in ORB's / LSD's left-image order
    std::vector<double> pt_disp, ls_sdisp, ls_edisp, ls_angle;          // [n], [m] x3
    std::vector<int32_t> pt_level, pt_src, ls_src;                       // [n] x2, [m]
    int frame_idx = 0;
    // results published by optimizePose (src/stereoFrameHandler.cpp:372-391), row-major
    std::array<double, 16> Tfw{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}, DT = Tfw;
    std::array<double, 36> Tfw_cov{}, DT_cov{};
    std::array<double, 6> DT_cov_eig{};
    double err_norm = -1.0;

    int n_pt() const { return (int)(pdesc.size() / 32); }
    int n_ls() const { return (int)(ldesc.size() / 32); }
    PlFrameBatch view(std::array<int32_t, 2>& pt_off, std::array<int32_t, 2>& ls_off) const {
        pt_off = {0, n_pt()};
        ls_off = {0, n_ls()};
        return PlFrameBatch{1, pt_off.data(), ls_off.data(), pdesc.data(), ldesc.data(), pt_P.data(), pt_pl.data(),
                            pt_sigma2.data(), ls_sP.data(), ls_eP.data(), ls_le.data(), ls_spl.data(), ls_epl.data(),
                            ls_sigma2.data(), ls_level.empty() ? nullptr : ls_level.data()};
    }
};

// matching.h surface (src/matching.cpp:41-91)
inline int matchNNR(Context& c, const std::vector<uint8_t>& d1, const std::vector<uint8_t>& d2, float nnr,
                    std::vector<int>& matches_12) {
    matches_12.assign(d1.size() / 32, -1);
    return c.check(plstvo_match_nnr(c.get(), d1.data(), (int)(d1.size() / 32), d2.data(), (int)(d2.size() / 32), 32, nnr,
                                    matches_12.data()));
}
inline int match(Context& c, const std::vector<uint8_t>& d1, const std::vector<uint8_t>& d2, float nnr,
                 bool best_lr_matches, std::vector<int>& matches_12) {
    matches_12.assign(d1.size() / 32, -1);
    return c.check(plstvo_match(c.get(), d1.data(), (int)(d1.size() / 32), d2.data(), (int)(d2.size() / 32), 32, nnr,
                                best_lr_matches ? 1 : 0, matches_12.data()));
}

// StereoFrame::matchStereoPoints / matchStereoLines (src/stereoFrame.cpp:120-173, :309-398) for one frame of raw stereo
// features: fills the frame's point / line records (and the compacted descriptor rows) exactly like the reference's loops.
struct KeyPoints {                       // cv::KeyPoint fields the step reads
    std::vector<float> pt;               // [n][2]
    std::vector<int32_t> octave;         // [n]
    std::vector<uint8_t> desc;           // [n][32]
    int size() const { return (int)(desc.size() / 32); }
};
struct KeyLines {                        // KeyLine fields the step reads
    std::vector<float> seg;              // [m][4] start / end point
    std::vector<float> angle;            // [m]
    std::vector<int32_t> octave;         // [m]
    std::vector<uint8_t> desc;           // [m][32]
    int size() const { return (int)(desc.size() / 32); }
};
inline int matchStereoPoints(Context& c, const PlCamera& cam, const PlStereoMatchConfig& mc, const PlStereoConfig& sc,
                             const KeyPoints& l, const KeyPoints& r, StereoFrame& out, std::vector<double>* disp = nullptr) {
    const int n = l.size();
    const int32_t lo[2] = {0, n}, ro[2] = {0, r.size()};
    std::vector<double> pl(2 * (size_t)n), d((size_t)n), P(3 * (size_t)n), s2((size_t)n);
    std::vector<int32_t> level((size_t)n), src((size_t)n);
    std::vector<uint8_t> desc(32 * (size_t)n);
    int32_t k = 0;
    c.check(plstvo_match_stereo_points(c.get(), &cam, &mc, &sc, 1, lo, l.pt.data(), l.octave.data(), l.desc.data(), ro, r.pt.data(),
                                       r.desc.data(), nullptr, pl.data(), d.data(), P.data(), s2.data(), level.data(), desc.data(),
                                       src.data(), &k));
    out.pt_pl.assign(pl.begin(), pl.begin() + 2 * (size_t)k);
    out.pt_P.assign(P.begin(), P.begin() + 3 * (size_t)k);
    out.pt_sigma2.assign(s2.begin(), s2.begin() + k);
    out.pdesc.assign(desc.begin(), desc.begin() + 32 * (size_t)k);
    if (disp) disp->assign(d.begin(), d.begin() + k);
    return k;
}
// ORB description after key-point selection (cv::ORB::compute; angle == nullptr: detectAndCompute's computed angles) for one
// grey image (row-major, width * height bytes).  kp.pt / kp.octave are read; kp is replaced by the survivors of the border
// filter, in input order, with their 32-byte descriptors, and angle (if given) likewise; returns the survivor count.
inline int computeORB(Context& c, const PlOrbConfig& cfg, const uint8_t* image, int width, int height, KeyPoints& kp,
                      std::vector<float>* angle = nullptr) {
    const int n = (int)(kp.pt.size() / 2);
    const int32_t off[2] = {0, n};
    std::vector<float> ang_out((size_t)n);
    std::vector<uint8_t> desc(32 * (size_t)n);
    std::vector<int32_t> src((size_t)n);
    const float* ang_in = (angle && (int)angle->size() == n) ? angle->data() : nullptr;
    const int k = c.check(plstvo_orb_compute_batch(c.get(), &cfg, 1, width, height, image, off, kp.pt.data(), kp.octave.data(),
                                                   ang_in, ang_out.data(), desc.data(), src.data(), nullptr));
    KeyPoints out;
    for (int i = 0; i < k; ++i) {
        out.pt.push_back(kp.pt[2 * (size_t)src[i]]);
        out.pt.push_back(kp.pt[2 * (size_t)src[i] + 1]);
        out.octave.push_back(kp.octave[src[i]]);
    }
    out.desc.assign(desc.begin(), desc.begin() + 32 * (size_t)k);
    kp = std::move(out);
    if (angle) angle->assign(ang_out.begin(), ang_out.begin() + k);
    return k;
}
// ORB::detectAndCompute on one grey image (row-major, width * height bytes), as StereoFrame::detectPointFeatures calls it
// (src/stereoFrame.cpp:104-118): fast_th != 0 replaces cfg.fast_threshold (the reference adapts it frame by frame, :109-111).
// kp is replaced by the key points, ordered by level, then y, then x on the level, with their descriptors; angle and response
// (if given) likewise.  Returns the key point count.
inline int detectAndComputeORB(Context& c, const PlOrbDetectConfig& cfg, const uint8_t* image, int width, int height,
                               KeyPoints& kp, int fast_th = 0, std::vector<float>* angle = nullptr,
                               std::vector<float>* response = nullptr) {
    const int32_t th = fast_th != 0 ? fast_th : cfg.fast_threshold;
    int cap = 2 * std::max(cfg.n_features, 0) + 64;
    std::vector<float> ang, resp;
    for (;;) {
        int32_t off[2] = {0, 0};
        kp.pt.resize(2 * (size_t)cap);
        kp.octave.resize((size_t)cap);
        kp.desc.resize(32 * (size_t)cap);
        ang.resize((size_t)cap);
        resp.resize((size_t)cap);
        const int rc = plstvo_orb_detect_and_compute_batch(c.get(), &cfg, 1, width, height, image, &th, cap, off, kp.pt.data(),
                                                           kp.octave.data(), ang.data(), resp.data(), kp.desc.data());
        if (rc == PLSTVO_E_TOO_LARGE && off[1] > cap && off[1] <= PLSTVO_MAX_FEATURES) {   // ties past the budget
            cap = off[1];
            continue;
        }
        const int n = c.check(rc);
        kp.pt.resize(2 * (size_t)n);
        kp.octave.resize((size_t)n);
        kp.desc.resize(32 * (size_t)n);
        if (angle) angle->assign(ang.begin(), ang.begin() + n);
        if (response) response->assign(resp.begin(), resp.begin() + n);
        return n;
    }
}
// LBD description of given octave-0 key lines (BinaryDescriptor::compute, default Params) on one grey image (row-major,
// width * height bytes), as StereoFrame::detectLineFeatures calls it after LSD (src/stereoFrame.cpp:242).  kl.seg (start
// and end point in the image) and kl.angle are read with num_pixels ([m] KeyLine::numOfPixels); kl.desc is replaced by the
// m descriptors, row i for line i.  Returns m; throws Error(PLSTVO_E_INVALID) when the three arrays do not describe the same
// m lines.
inline int computeLBD(Context& c, const uint8_t* image, int width, int height, KeyLines& kl,
                      const std::vector<int32_t>& num_pixels) {
    const int n = (int)(kl.seg.size() / 4);
    if (kl.seg.size() % 4 != 0 || kl.angle.size() != (size_t)n || num_pixels.size() != (size_t)n)
        throw Error(PLSTVO_E_INVALID, "computeLBD: kl.seg must hold 4 floats per line, kl.angle and num_pixels one entry per line");
    const int32_t off[2] = {0, n};
    std::vector<uint8_t> desc(32 * (size_t)n);
    const int k = c.check(plstvo_lbd_compute_batch(c.get(), 1, width, height, image, off, kl.seg.data(), kl.angle.data(),
                                                   num_pixels.data(), desc.data()));
    kl.desc = std::move(desc);
    return k;
}
// LSD key lines of one grey image (row-major, width * height bytes), as StereoFrame::detectLineFeatures detects them
// (src/stereoFrame.cpp:218-241) with llength_th = cfg.min_line_length * min(width, height), the product
// StereoFrameHandler computes (src/stereoFrameHandler.cpp:39).  kl.seg, kl.angle and kl.octave (all 0) are replaced by the
// key lines in the reference's order and kl.desc is cleared; num_pixels (what computeLBD takes), response and length (if
// given) likewise.  Returns the line count.
inline int detectLSD(Context& c, const PlLsdConfig& cfg, const uint8_t* image, int width, int height, KeyLines& kl,
                     std::vector<int32_t>& num_pixels, std::vector<float>* response = nullptr,
                     std::vector<float>* length = nullptr) {
    int cap = cfg.n_features > 0 ? cfg.n_features : 1024;
    std::vector<float> resp, len;
    for (;;) {
        int32_t off[2] = {0, 0};
        kl.seg.resize(4 * (size_t)cap);
        kl.angle.resize((size_t)cap);
        num_pixels.resize((size_t)cap);
        resp.resize((size_t)cap);
        len.resize((size_t)cap);
        const int rc = plstvo_lsd_detect_batch(c.get(), &cfg, 1, width, height, image, cap, off, kl.seg.data(), kl.angle.data(),
                                               num_pixels.data(), resp.data(), len.data());
        if (rc == PLSTVO_E_TOO_LARGE && off[1] > cap && off[1] <= PLSTVO_MAX_FEATURES) {   // more lines than the first guess
            cap = off[1];
            continue;
        }
        const int n = c.check(rc);
        kl.seg.resize(4 * (size_t)n);
        kl.angle.resize((size_t)n);
        kl.octave.assign((size_t)n, 0);
        kl.desc.clear();
        num_pixels.resize((size_t)n);
        if (response) response->assign(resp.begin(), resp.begin() + n);
        if (length) length->assign(len.begin(), len.begin() + n);
        return n;
    }
}
// The FLD branch's key lines of one width x height image (src/stereoFrame.cpp:260-299, plstvo_fld_key_lines): seg is
// FastLineDetector::detect's vector<Vec4f> as [n][4] floats, in its order; the caller ran
// createFastLineDetector(cfg.min_line_length * min(width, height)) on fld_img.  kl.seg, kl.angle and kl.octave (all 0) are
// replaced by the key lines in the reference's order and kl.desc is cleared; num_pixels, response and length (if given)
// likewise.  Host code.  Returns the line count.
inline int fldKeyLines(int width, int height, int n_features, const std::vector<float>& seg, KeyLines& kl,
                       std::vector<int32_t>& num_pixels, std::vector<float>* response = nullptr,
                       std::vector<float>* length = nullptr) {
    if (seg.size() % 4) throw Error(PLSTVO_E_INVALID, "fldKeyLines: seg must hold 4 floats per segment");
    const int n = (int)(seg.size() / 4), m = n_features > 0 ? std::min(n, n_features) : n;
    std::vector<float> resp((size_t)m), len((size_t)m);
    kl.seg.resize(4 * (size_t)m);
    kl.angle.resize((size_t)m);
    num_pixels.resize((size_t)m);
    const int k = plstvo_fld_key_lines(width, height, n_features, n, seg.data(), kl.seg.data(), kl.angle.data(),
                                       num_pixels.data(), resp.data(), len.data());
    if (k < 0) throw Error(k, "fldKeyLines: width or height outside 1..32767, or n_features < 0");
    kl.octave.assign((size_t)k, 0);
    kl.desc.clear();
    if (response) *response = std::move(resp);
    if (length) *length = std::move(len);
    return k;
}
// One stereo frame as StereoFrame::extractStereoFeatures starts it (src/stereoFrame.cpp:59-118, :182-243): the two grey images
// (row-major, width * height bytes each) and the key lines LSD kept on each (octave 0: start / end point [m][4], KeyLine::angle,
// KeyLine::numOfPixels).  fast_th 0: the config's FAST threshold.
struct StereoImageFrame {
    const uint8_t* img_l = nullptr;
    const uint8_t* img_r = nullptr;
    int32_t fast_th = 0;
    std::vector<float> seg_l, seg_r, angle_l, angle_r;
    std::vector<int32_t> npix_l, npix_r;
};
namespace detail {
struct StereoImagesPack {   // frames packed into the arrays a PlStereoImages points at
    std::vector<uint8_t> img_l, img_r;
    std::vector<int32_t> th, ll_off{0}, lr_off{0}, npix_l, npix_r;
    std::vector<float> seg_l, seg_r, angle_l, angle_r;
    PlStereoImages view{};
};
inline void packStereoImages(const std::vector<StereoImageFrame>& frames, int width, int height, StereoImagesPack& p) {
    const size_t px = (size_t)width * (size_t)height;
    for (const StereoImageFrame& f : frames) {
        const size_t nl = f.seg_l.size() / 4, nr = f.seg_r.size() / 4;
        if (!f.img_l || !f.img_r || f.seg_l.size() % 4 || f.seg_r.size() % 4 || f.angle_l.size() != nl || f.npix_l.size() != nl ||
            f.angle_r.size() != nr || f.npix_r.size() != nr)
            throw Error(PLSTVO_E_INVALID, "trackStereoImages: every frame needs both images, and seg (4 floats per line), angle and "
                                          "npix must describe the same lines on each side");
        p.img_l.insert(p.img_l.end(), f.img_l, f.img_l + px);
        p.img_r.insert(p.img_r.end(), f.img_r, f.img_r + px);
        p.th.push_back(f.fast_th);
        p.ll_off.push_back(p.ll_off.back() + (int32_t)nl);
        p.lr_off.push_back(p.lr_off.back() + (int32_t)nr);
        p.seg_l.insert(p.seg_l.end(), f.seg_l.begin(), f.seg_l.end());
        p.seg_r.insert(p.seg_r.end(), f.seg_r.begin(), f.seg_r.end());
        p.angle_l.insert(p.angle_l.end(), f.angle_l.begin(), f.angle_l.end());
        p.angle_r.insert(p.angle_r.end(), f.angle_r.begin(), f.angle_r.end());
        p.npix_l.insert(p.npix_l.end(), f.npix_l.begin(), f.npix_l.end());
        p.npix_r.insert(p.npix_r.end(), f.npix_r.begin(), f.npix_r.end());
    }
    p.view = PlStereoImages{(int32_t)frames.size(), width, height, p.img_l.data(), p.img_r.data(), p.th.data(), p.ll_off.data(),
                            p.lr_off.data(), p.seg_l.data(), p.seg_r.data(), p.angle_l.data(), p.angle_r.data(), p.npix_l.data(),
                            p.npix_r.data()};
}
// the view of images alone, for the calls that detect their own key lines: a frame that carries lines is rejected
inline void dropLines(const std::vector<StereoImageFrame>& frames, StereoImagesPack& p, const char* who) {
    for (const StereoImageFrame& f : frames)
        if (!f.seg_l.empty() || !f.seg_r.empty() || !f.angle_l.empty() || !f.angle_r.empty() || !f.npix_l.empty() ||
            !f.npix_r.empty())
            throw Error(PLSTVO_E_INVALID, std::string(who) + ": LSD runs inside the call, so frames must carry no key lines");
    p.view.ll_off = p.view.lr_off = nullptr;
    p.view.seg_l = p.view.seg_r = p.view.angle_l = p.view.angle_r = nullptr;
    p.view.npix_l = p.view.npix_r = nullptr;
}
}  // namespace detail
// ---- rectification: PinholeStereoCamera's maps (src/pinholeStereoCamera.cpp:30-182) and rectifyImagesLR (:196-208) ----
// One camera's CV_16SC2 + CV_16UC1 maps: map1 [height][width][2], map2 [height][width].
struct RectifyMaps {
    int width = 0, height = 0;
    std::vector<int16_t> map1;
    std::vector<uint16_t> map2;
};
// cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap with m1type CV_16SC2 (plstvo_init_undistort_rectify_map;
// host code, no GPU).
inline RectifyMaps initUndistortRectifyMap(const PlRectifyModel& model, int width, int height) {
    RectifyMaps m;
    m.width = width;
    m.height = height;
    const size_t px = width > 0 && height > 0 ? (size_t)width * (size_t)height : 1;
    m.map1.resize(2 * px);
    m.map2.resize(px);
    const int rc = plstvo_init_undistort_rectify_map(&model, width, height, m.map1.data(), m.map2.data());
    if (rc < 0) throw Error(rc, "initUndistortRectifyMap: unsupported model (coefficient count, singular P * R) or size");
    return m;
}
// A rig's maps resident in HBM (plstvo_rectifier_create); one map pair for both sides where only left is given.  The colour
// forms (plstvo_rectifier_create_color) take images of `channels` interleaved channels (3: BGR, 4: BGRA, as cv::imread
// gives them) and give the detectors cvtColor(remap(img), COLOR_BGR2GRAY), or without maps cvtColor alone.  Destroy it
// before its Context.
class Rectifier {
public:
    Rectifier(Context& c, const RectifyMaps& left, const RectifyMaps& right) : r_(create(c, 1, left, right)) {}
    Rectifier(Context& c, const RectifyMaps& both) : r_(create(c, 1, both, both)) {}
    Rectifier(Context& c, int channels, const RectifyMaps& left, const RectifyMaps& right)
        : r_(create(c, channels, left, right)), channels_(channels) {}
    Rectifier(Context& c, int channels, const RectifyMaps& both) : r_(create(c, channels, both, both)), channels_(channels) {}
    Rectifier(Context& c, int width, int height, int channels)
        : r_(check(c, plstvo_rectifier_create_color(c.get(), width, height, channels, nullptr, nullptr, nullptr, nullptr))),
          channels_(channels) {}
    ~Rectifier() { plstvo_rectifier_destroy(r_); }
    Rectifier(const Rectifier&) = delete;
    Rectifier& operator=(const Rectifier&) = delete;
    const PlRectifier* get() const { return r_; }
    int channels() const { return channels_; }   // bytes per pixel of the images it takes
private:
    static PlRectifier* check(Context& c, PlRectifier* p) {
        if (!p) throw Error(PLSTVO_E_INVALID, plstvo_last_error(c.get()));
        return p;
    }
    static PlRectifier* create(Context& c, int channels, const RectifyMaps& l, const RectifyMaps& r) {
        if (l.width != r.width || l.height != r.height) throw Error(PLSTVO_E_SIZE, "Rectifier: the two sides' maps differ in size");
        if (channels == 1)
            return check(c, plstvo_rectifier_create(c.get(), l.width, l.height, l.map1.data(), l.map2.data(), r.map1.data(),
                                                    r.map2.data()));
        return check(c, plstvo_rectifier_create_color(c.get(), l.width, l.height, channels, l.map1.data(), l.map2.data(),
                                                      r.map1.data(), r.map2.data()));
    }
    PlRectifier* r_ = nullptr;
    int channels_ = 1;
};
// PinholeStereoCamera::rectifyImagesLR on B pairs (plstvo_rectify_batch): out = cv::remap(img, maps, INTER_LINEAR), byte for
// byte; [B][height][width] grey in and out.  With a colour rectifier the input is [B][height][width][channels] and the output
// the grey image cvtColor(..., COLOR_BGR2GRAY) makes of it.
inline void rectifyImagesLR(Context& c, const Rectifier& r, const uint8_t* img_l, uint8_t* rec_l, const uint8_t* img_r,
                            uint8_t* rec_r, int B = 1) {
    c.check(plstvo_rectify_batch(c.get(), r.get(), B, img_l, img_r, rec_l, rec_r));
}
// The models and the rectified camera of each PinholeStereoCamera constructor branch.  stereoRectify is not built: the caller
// passes the R1 / R2 and P1 / P2 (3x4, row-major) that cv::stereoRectify(Kl, Dl, Kr, Dr, size, R, t, ..., CALIB_ZERO_DISPARITY,
// 0) gave, as the reference's constructor computes them.  cam: fx, fy, cx, cy from P1 and b = cam_bl, as given.
struct StereoRectification {
    PlRectifyModel left{}, right{};
    PlCamera cam{};
    bool one_map = false;   // the cam_d0 branch: the left map serves both sides

    // The Kl / Dl branch (EuRoC): K = (fx, fy, cx, cy) rounded to float as Mat_<float> stores it, D in double (4, 5 or 8
    // coefficients); equidistant: the dtype branch, cv::fisheye maps with 4 coefficients.
    static StereoRectification pinhole(int width, int height, double b, const double Kl[4], const std::vector<double>& Dl,
                                       const double Kr[4], const std::vector<double>& Dr, const double R1[9], const double P1[12],
                                       const double R2[9], const double P2[12], bool equidistant = false) {
        StereoRectification s;
        s.left = model(equidistant, Kl, Dl, R1, P1, true);
        s.right = model(equidistant, Kr, Dr, R2, P2, true);
        s.cam = camera(width, height, b, P1);
        return s;
    }
    // The cam_d0 branch (cam_d0 != 0): K, D (d0..d3, 0) and P in float, P's fy = fx, R = I; one map for both sides.
    static StereoRectification camD0(int width, int height, double fx, double fy, double cx, double cy, double b, double d0,
                                     double d1, double d2, double d3) {
        StereoRectification s;
        const double K[4] = {fx, fy, cx, cy};
        const double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        const double P[12] = {(float)fx, 0, (float)cx, 0, 0, (float)fx, (float)cy, 0, 0, 0, 1, 0};
        const std::vector<double> D{(float)d0, (float)d1, (float)d2, (float)d3, 0.0};
        s.left = s.right = model(false, K, D, R, P, true);
        s.cam = camera(width, height, b, P);
        s.one_map = true;
        return s;
    }
    // the maps of both sides, uploaded once; channels 3 or 4: a colour rectifier on these maps (images as cv::imread reads
    // KITTI's image_2 / image_3, or EuRoC's with IMREAD_UNCHANGED)
    Rectifier rectifier(Context& c, int channels = 1) const {
        const RectifyMaps l = initUndistortRectifyMap(left, cam.width, cam.height);
        if (one_map) return Rectifier(c, channels, l);
        return Rectifier(c, channels, l, initUndistortRectifyMap(right, cam.width, cam.height));
    }

private:
    static PlRectifyModel model(bool equidistant, const double K4[4], const std::vector<double>& D, const double R[9],
                                const double P[12], bool k_float) {
        PlRectifyModel m{};
        m.model = equidistant ? 1 : 0;
        m.n_dist = (double)D.size();
        auto kf = [k_float](double v) { return k_float ? (double)(float)v : v; };
        const double K[9] = {kf(K4[0]), 0, kf(K4[2]), 0, kf(K4[1]), kf(K4[3]), 0, 0, 1};
        std::copy(K, K + 9, m.K);
        std::copy(D.begin(), D.begin() + std::min<size_t>(D.size(), 8), m.D);
        std::copy(R, R + 9, m.R);
        std::copy(P, P + 12, m.P);
        return m;
    }
    static PlCamera camera(int width, int height, double b, const double P[12]) {
        PlCamera c{};
        c.fx = P[0]; c.fy = P[5]; c.cx = P[2]; c.cy = P[6]; c.b = b; c.width = width; c.height = height;
        return c;
    }
};

// Stereo images in, pose out (plstvo_track_stereo_images_batch): extractStereoFeatures with LSD left to the caller, then
// f2fTracking + optimizePose, for prev.size() independent (prev[p], curr[p]) pairs of images of cam's size.  priors: one per
// pair or empty (identity).  n_stereo (optional) receives [pairs][4] = stereo points, lines of prev, then of curr.
inline std::vector<PlPoseResult> trackStereoImages(Context& c, const PlCamera& cam, const PlConfig& cfg, const PlStereoMatchConfig& mc,
                                                   const PlStereoConfig& sc, const PlOrbDetectConfig& oc,
                                                   const std::vector<StereoImageFrame>& prev, const std::vector<StereoImageFrame>& curr,
                                                   const std::vector<PlPrior>& priors = {}, std::vector<int32_t>* n_stereo = nullptr) {
    if (prev.size() != curr.size()) throw Error(PLSTVO_E_SIZE, "trackStereoImages: prev and curr hold different numbers of frames");
    if (!priors.empty() && priors.size() != prev.size()) throw Error(PLSTVO_E_INVALID, "trackStereoImages: one prior per pair");
    detail::StereoImagesPack a, b;
    detail::packStereoImages(prev, cam.width, cam.height, a);
    detail::packStereoImages(curr, cam.width, cam.height, b);
    std::vector<PlPoseResult> res(std::max<size_t>(prev.size(), 1));
    std::vector<int32_t> ns(4 * prev.size());
    c.check(plstvo_track_stereo_images_batch(c.get(), &cam, &cfg, &mc, &sc, &oc, &a.view, &b.view,
                                             priors.empty() ? nullptr : priors.data(), res.data(), ns.data()));
    res.resize(prev.size());
    if (n_stereo) *n_stereo = std::move(ns);
    return res;
}
// The same for consecutive frames (plstvo_track_stereo_images_sequence): frames.size() - 1 results, pair p = (frame p, frame p + 1);
// every frame's images are detected and described once.  n_stereo (optional): [frames][2] = stereo points, lines per frame.
inline std::vector<PlPoseResult> trackStereoImageSequence(Context& c, const PlCamera& cam, const PlConfig& cfg,
                                                          const PlStereoMatchConfig& mc, const PlStereoConfig& sc,
                                                          const PlOrbDetectConfig& oc, const std::vector<StereoImageFrame>& frames,
                                                          const std::vector<PlPrior>& priors = {},
                                                          std::vector<int32_t>* n_stereo = nullptr) {
    const size_t pairs = frames.empty() ? 0 : frames.size() - 1;
    if (!priors.empty() && priors.size() != pairs) throw Error(PLSTVO_E_INVALID, "trackStereoImageSequence: one prior per pair");
    detail::StereoImagesPack a;
    detail::packStereoImages(frames, cam.width, cam.height, a);
    std::vector<PlPoseResult> res(std::max<size_t>(pairs, 1));   // the call takes a non-null results array even with no pair
    std::vector<int32_t> ns(2 * frames.size());
    c.check(plstvo_track_stereo_images_sequence(c.get(), &cam, &cfg, &mc, &sc, &oc, &a.view,
                                                priors.empty() ? nullptr : priors.data(), res.data(), ns.data()));
    res.resize(pairs);
    if (n_stereo) *n_stereo = std::move(ns);
    return res;
}
// Stereo images alone in, pose out (plstvo_track_stereo_images_lsd_batch): as trackStereoImages above, with LSD under lc run
// inside the call.  Every frame's line vectors must be empty (Error(PLSTVO_E_INVALID) otherwise).
inline std::vector<PlPoseResult> trackStereoImages(Context& c, const PlCamera& cam, const PlConfig& cfg, const PlStereoMatchConfig& mc,
                                                   const PlStereoConfig& sc, const PlOrbDetectConfig& oc, const PlLsdConfig& lc,
                                                   const std::vector<StereoImageFrame>& prev, const std::vector<StereoImageFrame>& curr,
                                                   const std::vector<PlPrior>& priors = {}, std::vector<int32_t>* n_stereo = nullptr) {
    if (prev.size() != curr.size()) throw Error(PLSTVO_E_SIZE, "trackStereoImages: prev and curr hold different numbers of frames");
    if (!priors.empty() && priors.size() != prev.size()) throw Error(PLSTVO_E_INVALID, "trackStereoImages: one prior per pair");
    detail::StereoImagesPack a, b;
    detail::packStereoImages(prev, cam.width, cam.height, a);
    detail::packStereoImages(curr, cam.width, cam.height, b);
    detail::dropLines(prev, a, "trackStereoImages");
    detail::dropLines(curr, b, "trackStereoImages");
    std::vector<PlPoseResult> res(std::max<size_t>(prev.size(), 1));
    std::vector<int32_t> ns(4 * prev.size());
    c.check(plstvo_track_stereo_images_lsd_batch(c.get(), &cam, &cfg, &mc, &sc, &oc, &lc, &a.view, &b.view,
                                                 priors.empty() ? nullptr : priors.data(), res.data(), ns.data()));
    res.resize(prev.size());
    if (n_stereo) *n_stereo = std::move(ns);
    return res;
}
// The same for consecutive frames (plstvo_track_stereo_images_lsd_sequence), as trackStereoImageSequence above.
inline std::vector<PlPoseResult> trackStereoImageSequence(Context& c, const PlCamera& cam, const PlConfig& cfg,
                                                          const PlStereoMatchConfig& mc, const PlStereoConfig& sc,
                                                          const PlOrbDetectConfig& oc, const PlLsdConfig& lc,
                                                          const std::vector<StereoImageFrame>& frames,
                                                          const std::vector<PlPrior>& priors = {},
                                                          std::vector<int32_t>* n_stereo = nullptr) {
    const size_t pairs = frames.empty() ? 0 : frames.size() - 1;
    if (!priors.empty() && priors.size() != pairs) throw Error(PLSTVO_E_INVALID, "trackStereoImageSequence: one prior per pair");
    detail::StereoImagesPack a;
    detail::packStereoImages(frames, cam.width, cam.height, a);
    detail::dropLines(frames, a, "trackStereoImageSequence");
    std::vector<PlPoseResult> res(std::max<size_t>(pairs, 1));
    std::vector<int32_t> ns(2 * frames.size());
    c.check(plstvo_track_stereo_images_lsd_sequence(c.get(), &cam, &cfg, &mc, &sc, &oc, &lc, &a.view,
                                                    priors.empty() ? nullptr : priors.data(), res.data(), ns.data()));
    res.resize(pairs);
    if (n_stereo) *n_stereo = std::move(ns);
    return res;
}
inline int matchStereoLines(Context& c, const PlCamera& cam, const PlStereoMatchConfig& mc, const PlStereoConfig& sc,
                            const KeyLines& l, const KeyLines& r, StereoFrame& out) {
    const int n = l.size();
    const int32_t lo[2] = {0, n}, ro[2] = {0, r.size()};
    const size_t N = (size_t)n;
    std::vector<double> spl(2 * N), epl(2 * N), sd(N), ed(N), sP(3 * N), eP(3 * N), le(3 * N), ang(N), s2(N);
    std::vector<int32_t> level(N), src(N);
    std::vector<uint8_t> desc(32 * N);
    int32_t k = 0;
    c.check(plstvo_match_stereo_lines(c.get(), &cam, &mc, &sc, 1, lo, l.seg.data(), l.angle.data(), l.octave.data(), l.desc.data(), ro,
                                      r.seg.data(), r.desc.data(), nullptr, spl.data(), epl.data(), sd.data(), ed.data(), sP.data(),
                                      eP.data(), le.data(), ang.data(), s2.data(), level.data(), desc.data(), src.data(), &k));
    const size_t K = (size_t)k;
    out.ls_spl.assign(spl.begin(), spl.begin() + 2 * K);
    out.ls_epl.assign(epl.begin(), epl.begin() + 2 * K);
    out.ls_sP.assign(sP.begin(), sP.begin() + 3 * K);
    out.ls_eP.assign(eP.begin(), eP.begin() + 3 * K);
    out.ls_le.assign(le.begin(), le.begin() + 3 * K);
    out.ls_sigma2.assign(s2.begin(), s2.begin() + K);
    out.ls_level.assign(level.begin(), level.begin() + K);
    out.ldesc.assign(desc.begin(), desc.begin() + 32 * K);
    return k;
}

// Host-side SE(3) helpers of the key-frame test (src/auxiliar.cpp:113-122, :143-173, :175-190), row-major arrays.
namespace se3 {
using Mat4 = std::array<double, 16>;
using Mat6 = std::array<double, 36>;
using Vec6 = std::array<double, 6>;

inline Mat4 identity4() { return Mat4{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; }
inline Mat4 mul(const Mat4& A, const Mat4& B) {
    Mat4 C{};
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc += A[4 * i + k] * B[4 * k + j];
            C[4 * i + j] = acc;
        }
    return C;
}
inline Mat4 inverse(const Mat4& T) {                     // inverse_se3: [R^T, -R^T t]
    Mat4 Ti = identity4();
    for (int i = 0; i < 3; ++i) {
        double acc = 0.0;
        for (int k = 0; k < 3; ++k) {
            Ti[4 * i + k] = T[4 * k + i];
            acc += -T[4 * k + i] * T[4 * k + 3];
        }
        Ti[4 * i + 3] = acc;
    }
    return Ti;
}
inline Vec6 logmap(const Mat4& T) {                      // logmap_se3: x = [V^-1 t ; w]
    double cosine = (T[0] + T[5] + T[10] - 1.0) / 2.0;
    if (cosine > 1.0) cosine = 1.0;                      // the reference's clamps: a NaN cosine stays NaN (theta NaN, w = 0)
    else if (cosine < -1.0) cosine = -1.0;
    double sine = std::sqrt(1.0 - cosine * cosine);
    if (sine > 1.0) sine = 1.0;
    else if (sine < -1.0) sine = -1.0;
    const double theta = std::acos(cosine);
    double w[3] = {0, 0, 0}, V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (theta > 0.000001) {
        const double k = theta / (2.0 * sine);
        w[0] = k * (T[9] - T[6]);                        // skewcoords(theta (R - R^T) / (2 sine))
        w[1] = k * (T[2] - T[8]);
        w[2] = k * (T[4] - T[1]);
        const double s[9] = {0, -w[2] / theta, w[1] / theta, w[2] / theta, 0, -w[0] / theta, -w[1] / theta, w[0] / theta, 0};
        const double a = (1.0 - cosine) / theta, b = (theta - sine) / theta;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double ss = 0.0;
                for (int m = 0; m < 3; ++m) ss += s[3 * i + m] * s[3 * m + j];
                V[3 * i + j] = (i == j ? 1.0 : 0.0) + s[3 * i + j] * a + ss * b;
            }
    }
    // V^-1 t by cofactors (Eigen's fixed 3x3 inverse)
    const double c00 = V[4] * V[8] - V[5] * V[7], c01 = V[5] * V[6] - V[3] * V[8], c02 = V[3] * V[7] - V[4] * V[6];
    const double det = V[0] * c00 + V[1] * c01 + V[2] * c02;
    const double inv[9] = {c00 / det, (V[2] * V[7] - V[1] * V[8]) / det, (V[1] * V[5] - V[2] * V[4]) / det,
                           c01 / det, (V[0] * V[8] - V[2] * V[6]) / det, (V[2] * V[3] - V[0] * V[5]) / det,
                           c02 / det, (V[1] * V[6] - V[0] * V[7]) / det, (V[0] * V[4] - V[1] * V[3]) / det};
    Vec6 x{};
    for (int i = 0; i < 3; ++i) {
        x[i] = inv[3 * i] * T[3] + inv[3 * i + 1] * T[7] + inv[3 * i + 2] * T[11];
        x[3 + i] = w[i];
    }
    return x;
}
inline Mat6 adjoint(const Mat4& T) {                     // adjoint_se3: [R, skew(t) R; 0, R]
    Mat6 A{};
    const double t[3] = {T[3], T[7], T[11]};
    const double sk[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            A[6 * i + j] = T[4 * i + j];
            A[6 * (i + 3) + j + 3] = T[4 * i + j];
            double acc = 0.0;
            for (int k = 0; k < 3; ++k) acc += sk[3 * i + k] * T[4 * k + j];
            A[6 * i + j + 3] = acc;
        }
    return A;
}
inline Mat6 sandwich(const Mat6& A, const Mat6& C) {     // A C A^T
    Mat6 AC{}, out{};
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 6; ++k) acc += A[6 * i + k] * C[6 * k + j];
            AC[6 * i + j] = acc;
        }
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 6; ++k) acc += AC[6 * i + k] * A[6 * j + k];
            out[6 * i + j] = acc;
        }
    return out;
}
inline Mat4 expmap(const Vec6& x) {                      // expmap_se3 (src/auxiliar.cpp:124-141): x = [t ; w]
    const double w[3] = {x[3], x[4], x[5]};
    const double theta = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {x[0], x[1], x[2]};
    if (!(theta < 0.000001)) {
        const double s[9] = {0, -w[2] / theta, w[1] / theta, w[2] / theta, 0, -w[0] / theta, -w[1] / theta, w[0] / theta, 0};
        double ss[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double acc = 0.0;
                for (int m = 0; m < 3; ++m) acc += s[3 * i + m] * s[3 * m + j];
                ss[3 * i + j] = acc;
            }
        const double sn = std::sin(theta), cs = std::cos(theta);
        double V[9];
        for (int k = 0; k < 9; ++k) {
            const double id = (k % 4 == 0) ? 1.0 : 0.0;
            R[k] = id + s[k] * sn + ss[k] * (1.0 - cs);
            V[k] = id + s[k] * (1.0 - cs) / theta + ss[k] * (theta - sn) / theta;
        }
        const double t0[3] = {t[0], t[1], t[2]};
        for (int i = 0; i < 3; ++i) t[i] = V[3 * i] * t0[0] + V[3 * i + 1] * t0[1] + V[3 * i + 2] * t0[2];
    }
    return Mat4{R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2], 0, 0, 0, 1};
}
inline Mat6 uncTinv(const Mat4& T, const Mat6& cov) { return sandwich(adjoint(inverse(T)), cov); }   // uncTinv_se3
inline double det6(Mat6 A) {                             // Matrix6d::determinant (partial-pivot LU, run to the end)
    double det = 1.0;
    for (int c = 0; c < 6; ++c) {
        int piv = c;
        for (int r = c + 1; r < 6; ++r)
            if (std::fabs(A[6 * r + c]) > std::fabs(A[6 * piv + c])) piv = r;
        if (piv != c) {
            for (int j = 0; j < 6; ++j) std::swap(A[6 * c + j], A[6 * piv + j]);
            det = -det;
        }
        det *= A[6 * c + c];
        if (A[6 * c + c] == 0.0) continue;               // a zero pivot skips its elimination; the product runs on
        for (int r = c + 1; r < 6; ++r) {
            const double f = A[6 * r + c] / A[6 * c + c];
            for (int j = c + 1; j < 6; ++j) A[6 * r + j] -= f * A[6 * c + j];
        }
    }
    return det;
}
}  // namespace se3

// Chains the per-pair results of plstvo_track_stereo_sequence (or of any batch of consecutive pairs solved with identity
// priors) into world poses exactly like optimizePose's tail does frame after frame (src/stereoFrameHandler.cpp:377-378, :388-389):
//   good pair: Tfw_k = expmap(logmap(Tfw_{k-1} DT_k)),  Tfw_cov_k = Tfw_cov_{k-1} + Ad(Tfw_{k-1}) DT_cov_k Ad(Tfw_{k-1})^T
//   failed   : Tfw_k = Tfw_{k-1},                       Tfw_cov_k = Tfw_cov_{k-1}
// Tfw0 / cov0: pose and covariance of the first frame (initialize(): identity, identity).  Writes results[k].Tfw / Tfw_cov.
inline void chainPoses(PlPoseResult* results, int n, se3::Mat4 Tfw0 = se3::identity4(), se3::Mat6 cov0 = [] {
                           se3::Mat6 c{};
                           for (int i = 0; i < 6; ++i) c[7 * i] = 1.0;
                           return c;
                       }()) {
    se3::Mat4 T = Tfw0;
    se3::Mat6 cov = cov0;
    for (int k = 0; k < n; ++k) {
        PlPoseResult& r = results[k];
        if (r.good) {
            se3::Mat4 DT;
            se3::Mat6 dc;
            std::copy(r.DT, r.DT + 16, DT.begin());
            std::copy(r.DT_cov, r.DT_cov + 36, dc.begin());
            const se3::Mat6 add = se3::sandwich(se3::adjoint(T), dc);
            for (int i = 0; i < 36; ++i) cov[i] += add[i];
            T = se3::expmap(se3::logmap(se3::mul(T, DT)));
        }
        std::copy(T.begin(), T.end(), r.Tfw);
        std::copy(cov.begin(), cov.end(), r.Tfw_cov);
    }
}

// The Config values of the handler's host-side state machine (adaptive FAST threshold, key-frame test):
// include/config.h:42-44, :56, :76-80, :100; defaults src/config.cpp:40-42, :52, :72-76, :102.
struct HandlerConfig {
    bool adaptative_fast = true;
    int fast_min_th = 5, fast_max_th = 50, fast_inc_th = 5, fast_feat_th = 50;
    float fast_err_th = 0.5f;
    int orb_fast_th = 20;
    double min_entropy_ratio = 0.85, max_kf_t_dist = 5.0, max_kf_r_dist = 15.0;
    // the adaptive threshold's values, as plstvo_stereo_session_run takes them
    PlHandlerConfig device() const {
        return PlHandlerConfig{adaptative_fast ? 1 : 0, fast_min_th, fast_max_th, fast_inc_th, fast_feat_th, fast_err_th};
    }
    // the key-frame test's values, as plstvo_stereo_session_run_keyframes takes them
    PlKeyframeConfig keyframes() const { return PlKeyframeConfig{min_entropy_ratio, max_kf_t_dist, max_kf_r_dist}; }
};

// StereoFrameHandler::updateFrame's adaptive FAST threshold (src/stereoFrameHandler.cpp:66-86): the threshold the caller's
// keypoint detector should use for the NEXT frame.
inline int updateFastThreshold(const HandlerConfig& c, int orb_fast_th, const StereoFrame& curr, int n_inliers_pt) {
    if (!c.adaptative_fast) return orb_fast_th;
    const int inc = c.fast_inc_th, feat = c.fast_feat_th;
    if (curr.DT == se3::identity4() || curr.err_norm > c.fast_err_th) return std::max(c.fast_min_th, orb_fast_th - 2 * inc);
    if (n_inliers_pt < feat) return std::max(c.fast_min_th, orb_fast_th - 2 * inc);
    if (n_inliers_pt < feat * 2) return std::max(c.fast_min_th, orb_fast_th - inc);
    if (n_inliers_pt > feat * 3) return std::min(c.fast_max_th, orb_fast_th + inc);
    return orb_fast_th;   // the reference's last branch (> 4 feat: + 2 inc, :84-85) is unreachable behind "> 3 feat"
}

// the identity 6x6 covariance that initialize and currFrameIsKF give a frame's Tfw_cov (src/stereoFrameHandler.cpp:45, :1195)
inline void identityCov(std::array<double, 36>& cov) {
    for (int i = 0; i < 36; ++i) cov[i] = (i % 7 == 0) ? 1.0 : 0.0;
}

// Key-frame test on the accumulated pose entropy (src/stereoFrameHandler.cpp:1136-1218; state include/stereoFrameHandler.h:81-86)
struct KeyframeTest {
    bool prev_f_iskf = true;
    double entropy_first_prevKF = 0.0;
    se3::Mat4 T_prevKF = se3::identity4();
    se3::Mat6 cov_prevKF_currF{};
    int N_prevKF_currF = 0;
    double entropy_curr = 0.0, entropy_ratio = 0.0, kf_t = 0.0, kf_r = 0.0;   // diagnostics of the last test

    bool needNewKF(const HandlerConfig& hcfg_, const StereoFrame& curr_frame) {   // :1136-1187
        const double k_entropy = 3.0 * (1.0 + std::log(2.0 * std::acos(-1.0)));
        if (prev_f_iskf) {                               // :1140-1153
            const double d = se3::det6(curr_frame.DT_cov);
            entropy_first_prevKF = (d != 0.0) ? k_entropy + 0.5 * std::log(d) : -999999999.99;
            prev_f_iskf = false;
        }
        const se3::Vec6 dX = se3::logmap(se3::mul(se3::inverse(curr_frame.Tfw), T_prevKF));   // :1156-1159
        kf_t = std::sqrt(dX[0] * dX[0] + dX[1] * dX[1] + dX[2] * dX[2]);
        kf_r = std::sqrt(dX[3] * dX[3] + dX[4] * dX[4] + dX[5] * dX[5]) * 180.f / 3.1415926535897932384626433832795;
        const se3::Mat6 add = se3::sandwich(se3::adjoint(T_prevKF), se3::uncTinv(curr_frame.DT, curr_frame.DT_cov));   // :1162-1164
        for (int i = 0; i < 36; ++i) cov_prevKF_currF[i] += add[i];
        entropy_curr = k_entropy + 0.5 * std::log(se3::det6(cov_prevKF_currF));
        entropy_ratio = entropy_curr / entropy_first_prevKF;
        bool zero_cov = true;
        for (double v : curr_frame.DT_cov) zero_cov = zero_cov && (v == 0.0);
        if (entropy_ratio < hcfg_.min_entropy_ratio || std::isnan(entropy_ratio) || std::isinf(entropy_ratio) ||
            (zero_cov && curr_frame.DT == se3::identity4()) || kf_t > hcfg_.max_kf_t_dist || kf_r > hcfg_.max_kf_r_dist ||
            N_prevKF_currF > 10)                         // :1173-1175
            return true;
        N_prevKF_currF++;
        return false;
    }
    // the state as plstvo_stereo_session_run_keyframes takes and returns it (the diagnostics are not part of it)
    PlKeyframeState state() const {
        PlKeyframeState s{};
        s.prev_f_iskf = prev_f_iskf ? 1 : 0;
        s.N_prevKF_currF = N_prevKF_currF;
        s.entropy_first_prevKF = entropy_first_prevKF;
        std::copy(T_prevKF.begin(), T_prevKF.end(), s.T_prevKF);
        std::copy(cov_prevKF_currF.begin(), cov_prevKF_currF.end(), s.cov_prevKF_currF);
        return s;
    }
    static KeyframeTest fromState(const PlKeyframeState& s) {
        KeyframeTest k;
        k.prev_f_iskf = s.prev_f_iskf != 0;
        k.N_prevKF_currF = s.N_prevKF_currF;
        k.entropy_first_prevKF = s.entropy_first_prevKF;
        std::copy(s.T_prevKF, s.T_prevKF + 16, k.T_prevKF.begin());
        std::copy(s.cov_prevKF_currF, s.cov_prevKF_currF + 36, k.cov_prevKF_currF.begin());
        return k;
    }
    void currFrameIsKF(StereoFrame& curr_frame) {        // :1189-1218 (feature idx renumbering is the caller's: dense order already)
        curr_frame.Tfw = se3::identity4();
        identityCov(curr_frame.Tfw_cov);
        T_prevKF = curr_frame.Tfw;
        cov_prevKF_currF.fill(0.0);
        prev_f_iskf = true;
        N_prevKF_currF = 0;
    }
};

// the prior optimizePose reads from prev_frame (src/stereoFrameHandler.cpp:317-326, :377-378)
inline PlPrior priorOf(const StereoFrame& prev_frame) {
    PlPrior prior;
    std::copy(prev_frame.Tfw.begin(), prev_frame.Tfw.end(), prior.Tfw);
    std::copy(prev_frame.Tfw_cov.begin(), prev_frame.Tfw_cov.end(), prior.Tfw_cov);
    std::copy(prev_frame.DT.begin(), prev_frame.DT.end(), prior.DT);
    std::copy(prev_frame.DT_cov.begin(), prev_frame.DT_cov.end(), prior.DT_cov);
    prior.err_norm = prev_frame.err_norm;
    return prior;
}
// optimizePose's results published into curr_frame (src/stereoFrameHandler.cpp:372-391)
inline void publishPose(const PlPoseResult& r, StereoFrame& curr_frame) {
    std::copy(r.DT, r.DT + 16, curr_frame.DT.begin());
    std::copy(r.DT_cov, r.DT_cov + 36, curr_frame.DT_cov.begin());
    std::copy(r.DT_cov_eig, r.DT_cov_eig + 6, curr_frame.DT_cov_eig.begin());
    std::copy(r.Tfw, r.Tfw + 16, curr_frame.Tfw.begin());
    std::copy(r.Tfw_cov, r.Tfw_cov + 36, curr_frame.Tfw_cov.begin());
    curr_frame.err_norm = r.err_norm;
}

// One stream's state of the reference's handler (include/stereoFrameHandler.h:56-86) and the steps on it that do not depend
// on how the frame reached the device: every handler below holds one per stream and drives it through these.
struct HandlerState {
    StereoFrame prev_frame, curr_frame;
    // the images handlers fill these with keepFeatures on only
    std::vector<int32_t> matches_pt, matches_ls;         // prev index -> curr index or -1
    std::vector<uint8_t> inlier_pt, inlier_ls;           // per prev feature: matched and still an inlier
    int n_inliers = 0, n_inliers_pt = 0, n_inliers_ls = 0;
    int orb_fast_th = 20;                                // include/stereoFrameHandler.h:62
    KeyframeTest kf;

    void initialize(const HandlerConfig& hcfg, StereoFrame frame) {   // src/stereoFrameHandler.cpp:35-52
        orb_fast_th = hcfg.orb_fast_th;                  // :38 (the threshold the first frame is detected with)
        prev_frame = std::move(frame);
        identityCov(prev_frame.Tfw_cov);
        kf = KeyframeTest{};                             // :48-51
    }
    void tracked(const PlPoseResult& r) {                // f2fTracking's matched counts (:126-128)
        n_inliers_pt = r.n_matched_pt;
        n_inliers_ls = r.n_matched_ls;
        n_inliers = n_inliers_pt + n_inliers_ls;
    }
    void optimizePose(const PlPoseResult& r) {           // :307-392: publish what the device computed
        publishPose(r, curr_frame);
        n_inliers_pt = r.n_inliers_pt;
        n_inliers_ls = r.n_inliers_ls;
        n_inliers = r.n_inliers;
    }
    void updateFrame(const HandlerConfig& hcfg) {        // :62-102
        orb_fast_th = updateFastThreshold(hcfg, orb_fast_th, curr_frame, n_inliers_pt);   // :66-86
        prev_frame = std::move(curr_frame);
        curr_frame = StereoFrame{};
    }
    // key-frame test (:1136-1218), PL-SLAM hooks: state in `kf`
    bool needNewKF(const HandlerConfig& hcfg) { return kf.needNewKF(hcfg, curr_frame); }
    void currFrameIsKF() { kf.currFrameIsKF(curr_frame); }
};

// StereoFrameHandler surface: initialize / insertStereoPair / optimizePose / updateFrame (app/imagesStVO.cpp:88-124)
class StereoFrameHandler : public HandlerState {
public:
    StereoFrameHandler(Context& ctx, const PlCamera& cam, const PlConfig& cfg, const HandlerConfig& hcfg = HandlerConfig{})
        : ctx_(ctx), cam_(cam), cfg_(cfg), hcfg_(hcfg) {}

    void initialize(StereoFrame frame) {                 // the caller extracts features with orb_fast_th from here on
        HandlerState::initialize(hcfg_, std::move(frame));
        has_prev_ = true;
    }
    void insertStereoPair(StereoFrame frame) {           // :54-60 (feature extraction is the caller's)
        if (!has_prev_) throw Error(PLSTVO_E_INVALID, "initialize() first");
        curr_frame = std::move(frame);
        f2fTracking();
    }
    void f2fTracking() {                                 // :106-129, fused with optimizePose on the device
        std::array<int32_t, 2> po1, lo1, po2, lo2;
        const PlFrameBatch prev = prev_frame.view(po1, lo1), curr = curr_frame.view(po2, lo2);
        const PlPrior prior = priorOf(prev_frame);
        matches_pt.assign(prev_frame.n_pt(), -1);
        matches_ls.assign(prev_frame.n_ls(), -1);
        inlier_pt.assign(prev_frame.n_pt(), 0);
        inlier_ls.assign(prev_frame.n_ls(), 0);
        ctx_.check(plstvo_track_batch(ctx_.get(), &cam_, &cfg_, &prev, &curr, &prior, &result_, matches_pt.data(),
                                      matches_ls.data(), inlier_pt.data(), inlier_ls.data()));
        tracked(result_);
    }
    void optimizePose() { HandlerState::optimizePose(result_); }
    void updateFrame() { HandlerState::updateFrame(hcfg_); }
    bool needNewKF() { return HandlerState::needNewKF(hcfg_); }
    const PlPoseResult& result() const { return result_; }

private:
    Context& ctx_;
    PlCamera cam_;
    PlConfig cfg_;
    HandlerConfig hcfg_;
    PlPoseResult result_{};
    bool has_prev_ = false;
};

// A PlStereoSession (plstvo_stereo_session_create): n_streams stereo streams, each stream's previous frame kept in HBM as its
// stereo features, so that a frame is detected and described once.  The configs are copied and fixed; rect (optional) must
// outlive the session.  Destroy it before its Context.
class StereoSession {
public:
    StereoSession(Context& c, const PlCamera& cam, const PlConfig& cfg, const PlStereoMatchConfig& mc, const PlStereoConfig& sc,
                  const PlOrbDetectConfig& oc, const PlLsdConfig& lc, int n_streams, const Rectifier* rect = nullptr)
        : c_(c), n_streams_(n_streams) {
        s_ = plstvo_stereo_session_create(c.get(), &cam, &cfg, &mc, &sc, &oc, &lc, rect ? rect->get() : nullptr, n_streams);
        if (!s_) throw Error(PLSTVO_E_INVALID, plstvo_last_error(c.get()));
    }
    // plstvo_stereo_session_create_cams: stream i tracked under cams[i] and prepared by rects[i] (rects empty: no stream is
    // remapped; a null entry in a grey session: that stream's images as given).  The rectifiers must outlive the session.
    StereoSession(Context& c, const std::vector<PlCamera>& cams, const PlConfig& cfg, const PlStereoMatchConfig& mc,
                  const PlStereoConfig& sc, const PlOrbDetectConfig& oc, const PlLsdConfig& lc,
                  const std::vector<const Rectifier*>& rects = {})
        : c_(c), n_streams_((int)cams.size()) {
        if (!rects.empty() && rects.size() != cams.size())
            throw Error(PLSTVO_E_INVALID, "StereoSession: one rectifier (or null) per camera");
        std::vector<const PlRectifier*> r;
        for (const Rectifier* x : rects) r.push_back(x ? x->get() : nullptr);
        s_ = plstvo_stereo_session_create_cams(c.get(), cams.data(), &cfg, &mc, &sc, &oc, &lc, r.empty() ? nullptr : r.data(),
                                               (int)cams.size());
        if (!s_) throw Error(PLSTVO_E_INVALID, plstvo_last_error(c.get()));
    }
    ~StereoSession() { plstvo_stereo_session_destroy(s_); }
    StereoSession(const StereoSession&) = delete;
    StereoSession& operator=(const StereoSession&) = delete;
    // initialize for streams ids[0 .. n): n_stereo [n][2] (optional)
    void initialize(int n, const int32_t* ids, const PlStereoImages& frames, int32_t* n_stereo = nullptr) {
        c_.check(plstvo_stereo_session_initialize(c_.get(), s_, n, ids, &frames, n_stereo));
    }
    // insertStereoPair + optimizePose for streams ids[0 .. n) against their kept frames: results [n], n_stereo [n][4] (optional)
    void insert(int n, const int32_t* ids, const PlStereoImages& frames, const PlPrior* priors, PlPoseResult* results,
                int32_t* n_stereo = nullptr) {
        c_.check(plstvo_stereo_session_insert(c_.get(), s_, n, ids, &frames, priors, results, n_stereo));
    }
    // plstvo_stereo_session_run: T steps of insert + optimizePose + updateFrame for streams ids[0 .. n), frames B = T * n
    // step-major; results [T][n], fast_th [T + 1][n] and n_stereo [T][n][4] optional
    void run(const PlHandlerConfig& h, int n, const int32_t* ids, int T, const PlStereoImages& frames, const int32_t* fast_th0,
             const PlPrior* priors, PlPoseResult* results, int32_t* fast_th = nullptr, int32_t* n_stereo = nullptr) {
        c_.check(plstvo_stereo_session_run(c_.get(), s_, &h, n, ids, T, &frames, fast_th0, priors, results, fast_th, n_stereo));
    }
    // plstvo_stereo_session_run_keyframes: run() with needNewKF / currFrameIsKF per stream and step; kf_state [n] in / out,
    // kf [T][n]
    void runKeyframes(const PlHandlerConfig& h, const PlKeyframeConfig& k, int n, const int32_t* ids, int T,
                      const PlStereoImages& frames, const int32_t* fast_th0, const PlPrior* priors, PlKeyframeState* kf_state,
                      PlPoseResult* results, PlKeyframeResult* kf, int32_t* fast_th = nullptr, int32_t* n_stereo = nullptr) {
        c_.check(plstvo_stereo_session_run_keyframes(c_.get(), s_, &h, &k, n, ids, T, &frames, fast_th0, priors, kf_state,
                                                     results, kf, fast_th, n_stereo));
    }
    // plstvo_stereo_session_run_schedule: run() / runKeyframes() over uneven streams; schedule [T][n] (0 idle, 1 insert,
    // 2 initialize), frames one per non-zero entry step-major; k null runs no key-frame test (kf_state, kf null)
    void runSchedule(const PlHandlerConfig& h, const PlKeyframeConfig* k, int n, const int32_t* ids, int T,
                     const uint8_t* schedule, const PlStereoImages& frames, const int32_t* fast_th0, const PlPrior* priors,
                     PlKeyframeState* kf_state, PlPoseResult* results, PlKeyframeResult* kf = nullptr,
                     int32_t* fast_th = nullptr, int32_t* n_stereo = nullptr) {
        c_.check(plstvo_stereo_session_run_schedule(c_.get(), s_, &h, k, n, ids, T, schedule, &frames, fast_th0, priors, kf_state,
                                                    results, kf, fast_th, n_stereo));
    }
    // plstvo_stereo_session_use_fld_lines: the reference's FLD line branch, before any stream is initialised.  On, every call
    // takes each frame's key lines in frames' key-line fields (fldKeyLines' rows; step-major for run / runKeyframes) and
    // LSD does not run.
    void useFLDLines(bool on) { c_.check(plstvo_stereo_session_use_fld_lines(c_.get(), s_, on ? 1 : 0)); }
    // plstvo_stereo_session_retain: keep each following call's frames and matches for read() (off frees them)
    void retain(bool on) { c_.check(plstvo_stereo_session_retain(c_.get(), s_, on ? 1 : 0)); }
    // plstvo_stereo_session_plot: draw each following initialize / insert's plotStereoFrame images for readPlot() (retention
    // must be on; off frees them)
    void plot(bool on) { c_.check(plstvo_stereo_session_plot(c_.get(), s_, on ? 1 : 0)); }
    // plstvo_stereo_session_read_plot of the last initialize / insert: n images of [height][width][3] BGR bytes into out,
    // sized from that call's n; returns n
    int readPlot(int n, int width, int height, std::vector<uint8_t>& out) const {
        out.resize((size_t)std::max(n, 1) * width * height * 3);
        if (c_.check(plstvo_stereo_session_read_plot(c_.get(), s_, out.data())) != n)
            throw Error(PLSTVO_E_INVALID, "StereoSession::readPlot: n differs from the last call's");
        out.resize((size_t)n * width * height * 3);
        return n;
    }
    // plstvo_stereo_session_read of the last call, into out's vectors sized from that call's n and n_stereo ([n][2] after an
    // initialize, [n][4] after an insert, as the call wrote it); out.m12_* / inlier_* are emptied after an initialize
    struct Frames {
        std::vector<double> pt_pl, pt_disp, pt_P, pt_sigma2;                                  // [N][2], [N], [N][3], [N]
        std::vector<int32_t> pt_level, pt_src;                                                // [N] x2
        std::vector<uint8_t> pdesc;                                                           // [N][32]
        std::vector<double> ls_spl, ls_epl, ls_sdisp, ls_edisp, ls_sP, ls_eP, ls_le, ls_angle, ls_sigma2;
        std::vector<int32_t> ls_level, ls_src;                                                // [M] x2
        std::vector<uint8_t> ldesc;                                                           // [M][32]
        std::vector<int32_t> m12_pt, m12_ls;                                                  // [kept points], [kept lines]
        std::vector<uint8_t> inlier_pt, inlier_ls;
        // The 19 lifted arrays, once, in PlStereoFrameOut's field order: f(this struct's member, StereoFrame's,
        // PlStereoFrameOut's, values per row, point (true) or line array) for each
        template <typename F> static void records(F&& f) {
            f(&Frames::pt_pl, &StereoFrame::pt_pl, &PlStereoFrameOut::pt_pl, 2, true);
            f(&Frames::pt_disp, &StereoFrame::pt_disp, &PlStereoFrameOut::pt_disp, 1, true);
            f(&Frames::pt_P, &StereoFrame::pt_P, &PlStereoFrameOut::pt_P, 3, true);
            f(&Frames::pt_sigma2, &StereoFrame::pt_sigma2, &PlStereoFrameOut::pt_sigma2, 1, true);
            f(&Frames::pt_level, &StereoFrame::pt_level, &PlStereoFrameOut::pt_level, 1, true);
            f(&Frames::pdesc, &StereoFrame::pdesc, &PlStereoFrameOut::pdesc, 32, true);
            f(&Frames::pt_src, &StereoFrame::pt_src, &PlStereoFrameOut::pt_src, 1, true);
            f(&Frames::ls_spl, &StereoFrame::ls_spl, &PlStereoFrameOut::ls_spl, 2, false);
            f(&Frames::ls_epl, &StereoFrame::ls_epl, &PlStereoFrameOut::ls_epl, 2, false);
            f(&Frames::ls_sdisp, &StereoFrame::ls_sdisp, &PlStereoFrameOut::ls_sdisp, 1, false);
            f(&Frames::ls_edisp, &StereoFrame::ls_edisp, &PlStereoFrameOut::ls_edisp, 1, false);
            f(&Frames::ls_sP, &StereoFrame::ls_sP, &PlStereoFrameOut::ls_sP, 3, false);
            f(&Frames::ls_eP, &StereoFrame::ls_eP, &PlStereoFrameOut::ls_eP, 3, false);
            f(&Frames::ls_le, &StereoFrame::ls_le, &PlStereoFrameOut::ls_le, 3, false);
            f(&Frames::ls_angle, &StereoFrame::ls_angle, &PlStereoFrameOut::ls_angle, 1, false);
            f(&Frames::ls_sigma2, &StereoFrame::ls_sigma2, &PlStereoFrameOut::ls_sigma2, 1, false);
            f(&Frames::ls_level, &StereoFrame::ls_level, &PlStereoFrameOut::ls_level, 1, false);
            f(&Frames::ldesc, &StereoFrame::ldesc, &PlStereoFrameOut::ldesc, 32, false);
            f(&Frames::ls_src, &StereoFrame::ls_src, &PlStereoFrameOut::ls_src, 1, false);
        }
    };
    void read(int n, const int32_t* n_stereo, bool insert, Frames& out) const {
        const PlStereoFrameOut o = outputs(n, n_stereo, insert, out);
        if (c_.check(plstvo_stereo_session_read(c_.get(), s_, &o)) != n)
            throw Error(PLSTVO_E_INVALID, "StereoSession::read: n differs from the last call's");
    }
    // plstvo_stereo_session_run_keyframes' key frames (retention on) into out's point and line vectors; rows [n_kf][4]: step,
    // stream id, points, lines.  out.m12_* / inlier_* are emptied.
    void readKeyframes(Frames& out, std::vector<int32_t>& rows) const {
        PlStereoFrameOut none{};
        const int n_kf = c_.check(plstvo_stereo_session_read_keyframes(c_.get(), s_, &none, nullptr));
        rows.assign(4 * (size_t)n_kf, 0);
        c_.check(plstvo_stereo_session_read_keyframes(c_.get(), s_, &none, rows.data()));
        std::vector<int32_t> ns(2 * (size_t)n_kf, 0);   // as an initialize's n_stereo: points, lines
        for (int j = 0; j < n_kf; ++j) {
            ns[2 * (size_t)j] = rows[4 * (size_t)j + 2];
            ns[2 * (size_t)j + 1] = rows[4 * (size_t)j + 3];
        }
        const PlStereoFrameOut o = outputs(n_kf, ns.data(), false, out);
        if (c_.check(plstvo_stereo_session_read_keyframes(c_.get(), s_, &o, nullptr)) != n_kf)
            throw Error(PLSTVO_E_INVALID, "StereoSession::readKeyframes: the number of key frames changed");
    }
    int streams() const { return n_streams_; }
    int64_t deviceBytes() const { return plstvo_stereo_session_device_bytes(s_); }
    PlStereoSession* get() const { return s_; }
private:
    // out's vectors sized for n frames of n_stereo ([n][4] with insert, else [n][2]; the tracker's rows with insert only)
    static PlStereoFrameOut outputs(int n, const int32_t* n_stereo, bool insert, Frames& out) {
        const int cols = insert ? 4 : 2;
        size_t np = 0, nl = 0, kp = 0, kl = 0;
        for (int k = 0; k < n; ++k) {
            np += (size_t)n_stereo[cols * k + cols - 2];
            nl += (size_t)n_stereo[cols * k + cols - 1];
            if (insert) {
                kp += (size_t)n_stereo[cols * k];
                kl += (size_t)n_stereo[cols * k + 1];
            }
        }
        PlStereoFrameOut o{};
        Frames::records([&](auto frames, auto, auto field, size_t per_row, bool point) {
            (out.*frames).resize(per_row * (point ? np : nl));
            o.*field = (out.*frames).data();
        });
        out.m12_pt.assign(kp, -1); out.m12_ls.assign(kl, -1); out.inlier_pt.assign(kp, 0); out.inlier_ls.assign(kl, 0);
        o.m12_pt = out.m12_pt.data(); o.inlier_pt = out.inlier_pt.data();
        o.m12_ls = out.m12_ls.data(); o.inlier_ls = out.inlier_ls.data();
        return o;
    }
    Context& c_;
    PlStereoSession* s_ = nullptr;
    int n_streams_ = 0;
};

namespace detail {
// A StereoSession::read (or readKeyframes) taken apart in call order: each call takes the next frame's rows.
struct ReadCursor {
    const StereoSession::Frames& r;
    size_t p0 = 0, l0 = 0, kp0 = 0, kl0 = 0;   // rows taken: points, lines, then the tracker's kept points, lines

    // the next frame's np points and nl lines into f's feature arrays
    void frameFromRead(size_t np, size_t nl, StereoFrame& f) {
        StereoSession::Frames::records([&](auto frames, auto frame, auto, size_t per_row, bool point) {
            const auto& src = r.*frames;
            const size_t first = point ? p0 : l0, count = point ? np : nl;
            (f.*frame).assign(src.begin() + (std::ptrdiff_t)(first * per_row),
                              src.begin() + (std::ptrdiff_t)((first + count) * per_row));
        });
        p0 += np;
        l0 += nl;
    }
    // the next kept frame's tracker rows (kp points, kl lines) into s's matches and inlier flags
    void tracked(size_t kp, size_t kl, HandlerState& s) {
        auto cut = [](auto& dst, const auto& src, size_t first, size_t count) {
            dst.assign(src.begin() + (std::ptrdiff_t)first, src.begin() + (std::ptrdiff_t)(first + count));
        };
        cut(s.matches_pt, r.m12_pt, kp0, kp);
        cut(s.inlier_pt, r.inlier_pt, kp0, kp);
        cut(s.matches_ls, r.m12_ls, kl0, kl);
        cut(s.inlier_ls, r.inlier_ls, kl0, kl);
        kp0 += kp;
        kl0 += kl;
    }
};
// One call's StereoSession::read split into its streams, given in call order: stream k's `frame` takes frame k's rows and,
// after an insert (n_stereo of 4 columns, else 2), its matches_pt / _ls and inlier_pt / _ls its kept frame's tracker rows.
inline void splitRead(const StereoSession::Frames& r, const int32_t* n_stereo, int cols,
                      const std::vector<HandlerState*>& streams, StereoFrame HandlerState::*frame) {
    ReadCursor c{r};
    for (size_t k = 0; k < streams.size(); ++k) {
        const int32_t* ns = n_stereo + cols * k;
        c.frameFromRead((size_t)ns[cols - 2], (size_t)ns[cols - 1], streams[k]->*frame);
        if (cols == 4) c.tracked((size_t)ns[0], (size_t)ns[1], *streams[k]);
    }
}
}  // namespace detail

namespace detail {
// n frames of one size (channels bytes per pixel), copied into the contiguous arrays a PlStereoImages of images alone points at
struct StereoImagesBatch {
    std::vector<uint8_t> img_l, img_r;
    std::vector<int32_t> th;
    PlStereoImages view{};
    void pack(int width, int height, int channels, const std::vector<const uint8_t*>& l, const std::vector<const uint8_t*>& r,
              const std::vector<int32_t>& fast_th, const char* who) {
        const size_t px = (size_t)width * (size_t)height * (size_t)channels, n = l.size();
        if (r.size() != n || fast_th.size() != n) throw Error(PLSTVO_E_INVALID, std::string(who) + ": ids and images differ in number");
        img_l.resize(n * px);
        img_r.resize(n * px);
        for (size_t k = 0; k < n; ++k) {
            if (!l[k] || !r[k]) throw Error(PLSTVO_E_INVALID, std::string(who) + ": null image");
            std::copy(l[k], l[k] + px, img_l.begin() + k * px);
            std::copy(r[k], r[k] + px, img_r.begin() + k * px);
        }
        th = fast_th;
        view = PlStereoImages{(int32_t)n, width, height, img_l.data(), img_r.data(), th.data()};
    }
    // the FLD branch's key lines of the packed frames: image k's FastLineDetector segments seg_l[k] / seg_r[k] ([m][4] floats,
    // FLD's order) through fldKeyLines, into the view's key-line fields
    std::vector<int32_t> ll_off, lr_off, npix_l, npix_r;
    std::vector<float> seg_l, seg_r, angle_l, angle_r;
    void addFLDLines(int width, int height, int n_features, const std::vector<std::vector<float>>& fl,
                     const std::vector<std::vector<float>>& fr, const char* who) {
        if (fl.size() != (size_t)view.B || fr.size() != (size_t)view.B)
            throw Error(PLSTVO_E_INVALID, std::string(who) + ": one segment list per image");
        ll_off.assign(1, 0); lr_off.assign(1, 0);
        npix_l.clear(); npix_r.clear(); seg_l.clear(); seg_r.clear(); angle_l.clear(); angle_r.clear();
        KeyLines kl;
        std::vector<int32_t> npix;
        for (size_t k = 0; k < fl.size(); ++k)
            for (int side = 0; side < 2; ++side) {
                fldKeyLines(width, height, n_features, (side ? fr : fl)[k], kl, npix);
                std::vector<int32_t>& off = side ? lr_off : ll_off;
                off.push_back(off.back() + (int32_t)npix.size());
                (side ? seg_r : seg_l).insert((side ? seg_r : seg_l).end(), kl.seg.begin(), kl.seg.end());
                (side ? angle_r : angle_l).insert((side ? angle_r : angle_l).end(), kl.angle.begin(), kl.angle.end());
                (side ? npix_r : npix_l).insert((side ? npix_r : npix_l).end(), npix.begin(), npix.end());
            }
        view.ll_off = ll_off.data(); view.lr_off = lr_off.data();
        view.seg_l = seg_l.data(); view.seg_r = seg_r.data();
        view.angle_l = angle_l.data(); view.angle_r = angle_r.data();
        view.npix_l = npix_l.data(); view.npix_r = npix_r.data();
    }
};
// the handler's ORB config: a frame's fast_th of 0 stands for the config's threshold; with that set to 0 too, every frame is
// detected with the threshold the handler chose, 0 included (updateFastThreshold returns 0 when fast_min_th <= 0), as in the
// reference
inline PlOrbDetectConfig handlerOrbConfig(PlOrbDetectConfig oc) {
    oc.fast_threshold = 0;
    return oc;
}
}  // namespace detail

// The same surface over images alone, as app/imagesStVO.cpp:88-97 drives the reference's handler: initialize(img_l, img_r, idx)
// and insertStereoPair(img_l, img_r, idx) take two grey images of cam's size (row-major, width * height bytes each), then
// optimizePose(), updateFrame() (with updateFastThreshold), needNewKF() and currFrameIsKF() as above.  It runs on a session
// of one stream: initialize detects the frame at orb_fast_th and keeps its stereo features on the device; each
// insertStereoPair is one plstvo_stereo_session_insert, which detects and describes the new images only, tracks them against
// the kept frame with the prior f2fTracking builds from prev_frame, and keeps the new frame in its place.  The results equal
// those of plstvo_track_stereo_raw_images_batch on (previous images, new images), byte for byte.  As in the reference's loop,
// updateFrame follows each insertStereoPair: the device already holds the new frame as the previous one.  prev_frame /
// curr_frame hold the pose state; their feature arrays stay empty unless keepFeatures(true) is on.  Then initialize fills
// prev_frame's arrays and insertStereoPair curr_frame's, with matches_pt / _ls and inlier_pt / _ls as StereoFrameHandler
// has them, all read back from the device after the call (StereoSession::read): such a frame can be given to the
// features-in StereoFrameHandler as it is.
class StereoImageHandler : public HandlerState {
public:
    StereoImageHandler(Context& ctx, const PlCamera& cam, const PlConfig& cfg, const PlStereoMatchConfig& mc,
                       const PlStereoConfig& sc, const PlOrbDetectConfig& oc, const PlLsdConfig& lc,
                       const HandlerConfig& hcfg = HandlerConfig{})
        : cam_(cam), hcfg_(hcfg), session_(ctx, cam, cfg, mc, sc, detail::handlerOrbConfig(oc), lc, 1) {}
    // Raw images, as Dataset::nextFrame feeds the reference's handler (src/dataset.cpp:147-157): initialize / insertStereoPair
    // take the camera's images before rectifyImagesLR, and each call rectifies them on the device under rect; cam is the
    // rectified camera (StereoRectification::cam).  With a colour rectifier the images are [height][width][channels] (BGR or
    // BGRA, as cv::imread gives them) and are converted to grey on the device after the remap.  rect must outlive the handler.
    StereoImageHandler(Context& ctx, const Rectifier& rect, const PlCamera& cam, const PlConfig& cfg, const PlStereoMatchConfig& mc,
                       const PlStereoConfig& sc, const PlOrbDetectConfig& oc, const PlLsdConfig& lc,
                       const HandlerConfig& hcfg = HandlerConfig{})
        : cam_(cam), hcfg_(hcfg), session_(ctx, cam, cfg, mc, sc, detail::handlerOrbConfig(oc), lc, 1, &rect) {}

    void initialize(const uint8_t* img_l, const uint8_t* img_r, int idx = 0) {   // src/stereoFrameHandler.cpp:35-52
        // :38, set here already because images() takes the first frame's threshold from it; HandlerState::initialize sets
        // the same value again below
        orb_fast_th = hcfg_.orb_fast_th;
        images(img_l, img_r);
        const int32_t id = 0;
        int32_t ns[2] = {0, 0};
        session_.initialize(1, &id, frame_, ns);
        frame_ = PlStereoImages{};
        StereoFrame frame;
        frame.frame_idx = idx;
        // resets prev_frame and kf before the read below: should that read throw, kf is reset already (prev_frame would be
        // reset either way, as the device already holds the new frame)
        HandlerState::initialize(hcfg_, std::move(frame));
        if (keep_) {
            session_.read(1, ns, false, read_);
            detail::splitRead(read_, ns, 2, {this}, &HandlerState::prev_frame);
        }
        if (plot_) session_.readPlot(1, cam_.width, cam_.height, plot_img_);
        has_prev_ = true;
    }
    // keep each frame's stereo features and the matches on the host after every call (off by default); effective from the
    // next initialize / insertStereoPair
    void keepFeatures(bool on) {
        session_.retain(on || plot_);   // plotting draws the retained rows
        keep_ = on;
    }
    // draw each new frame's plotStereoFrame() image on the device after every call (off by default); effective from the next
    // initialize / insertStereoPair
    void plotFrames(bool on) {
        if (on) session_.retain(true);
        session_.plot(on);
        if (!on && !keep_) session_.retain(false);
        plot_ = on;
        plot_img_.clear();
    }
    // StereoFrame::plotStereoFrame() of the frame the last initialize / insertStereoPair produced, as app/imagesStVO.cpp:109
    // hands it to its scene: [height][width][3] BGR bytes, the rectified left image with the stereo points' circles and the
    // stereo lines in (0, 200, 0).  Empty with plotFrames off.
    const std::vector<uint8_t>& plotStereoFrame() const { return plot_img_; }
    void insertStereoPair(const uint8_t* img_l, const uint8_t* img_r, int idx = 0) {   // :54-60
        if (!has_prev_) throw Error(PLSTVO_E_INVALID, "initialize() first");
        images(img_l, img_r);
        curr_frame = StereoFrame{};
        curr_frame.frame_idx = idx;
        f2fTracking();
    }
    void f2fTracking() {                                 // :106-129, with the new frame's feature extraction, fused with optimizePose
        if (!frame_.img_l) throw Error(PLSTVO_E_INVALID, "insertStereoPair() first");
        const PlPrior prior = priorOf(prev_frame);
        const int32_t id = 0;
        const PlStereoImages f = frame_;
        frame_ = PlStereoImages{};
        session_.insert(1, &id, f, &prior, &result_, n_stereo.data());
        if (keep_) {
            session_.read(1, n_stereo.data(), true, read_);
            detail::splitRead(read_, n_stereo.data(), 4, {this}, &HandlerState::curr_frame);
        }
        if (plot_) session_.readPlot(1, cam_.width, cam_.height, plot_img_);
        tracked(result_);
    }
    void optimizePose() { HandlerState::optimizePose(result_); }
    void updateFrame() { HandlerState::updateFrame(hcfg_); }
    bool needNewKF() { return HandlerState::needNewKF(hcfg_); }
    const PlPoseResult& result() const { return result_; }

    std::array<int32_t, 4> n_stereo{};                   // stereo points, lines of prev, then of curr, in the last call

private:
    // the caller's images for the next session call, detected at orb_fast_th (they are read during that call only)
    void images(const uint8_t* img_l, const uint8_t* img_r) {
        if (!img_l || !img_r) throw Error(PLSTVO_E_INVALID, "StereoImageHandler: null image");
        th_ = orb_fast_th;
        frame_ = PlStereoImages{1, cam_.width, cam_.height, img_l, img_r, &th_};
    }
    PlCamera cam_;
    HandlerConfig hcfg_;
    StereoSession session_;
    PlPoseResult result_{};
    PlStereoImages frame_{};
    int32_t th_ = 0;
    bool has_prev_ = false;
    bool keep_ = false;
    bool plot_ = false;
    std::vector<uint8_t> plot_img_;
    StereoSession::Frames read_;
};

// Many StereoImageHandlers at once: one per stream (camera) of a session, each with the reference handler's state, and one
// session call per initialize / insertStereoPairs over any subset of the streams.  Stream k behaves exactly as a
// StereoImageHandler fed only stream k's images: the same thresholds (updateFastThreshold), priors (priorOf), poses and
// key-frame test.  Streams need not run in lockstep; a stream not named keeps its frame and state.  Per named stream, as the
// reference's loop: insertStereoPairs, then optimizePose, needNewKF / currFrameIsKF if wanted, and updateFrame.
class StereoStreamsHandler {
public:
    struct Stream : HandlerState {
        std::array<int32_t, 4> n_stereo{};               // stereo points, lines of prev, then of curr, in the stream's last insert
        PlPoseResult result{};
        bool has_prev = false;
        std::vector<uint8_t> plot;                       // plotFrames: the image of the stream's last initialize / insert
    };
    StereoStreamsHandler(Context& ctx, const PlCamera& cam, const PlConfig& cfg, const PlStereoMatchConfig& mc,
                         const PlStereoConfig& sc, const PlOrbDetectConfig& oc, const PlLsdConfig& lc, int n_streams,
                         const HandlerConfig& hcfg = HandlerConfig{}, const Rectifier* rect = nullptr)
        : cam_(cam), hcfg_(hcfg), session_(ctx, cam, cfg, mc, sc, detail::handlerOrbConfig(oc), lc, n_streams, rect),
          streams_((size_t)n_streams), channels_(rect ? rect->channels() : 1), lsd_nfeatures_(lc.n_features),
          has_lines_(cfg.has_lines != 0) {
        for (Stream& s : streams_) s.orb_fast_th = hcfg_.orb_fast_th;
    }
    // One camera per stream, as one PinholeStereoCamera per StereoFrameHandler in the reference, and optionally one rectifier
    // per stream (StereoSession's cams constructor).  The cameras share one image size.
    StereoStreamsHandler(Context& ctx, const std::vector<PlCamera>& cams, const PlConfig& cfg, const PlStereoMatchConfig& mc,
                         const PlStereoConfig& sc, const PlOrbDetectConfig& oc, const PlLsdConfig& lc,
                         const HandlerConfig& hcfg = HandlerConfig{}, const std::vector<const Rectifier*>& rects = {})
        : cam_(cams.at(0)), hcfg_(hcfg), session_(ctx, cams, cfg, mc, sc, detail::handlerOrbConfig(oc), lc, rects),
          streams_(cams.size()), lsd_nfeatures_(lc.n_features), has_lines_(cfg.has_lines != 0) {
        for (const Rectifier* r : rects)
            if (r) {
                channels_ = r->channels();
                break;
            }
        for (Stream& s : streams_) s.orb_fast_th = hcfg_.orb_fast_th;
    }

    // The reference's FLD line branch (use_fld_lines, StereoSession::useFLDLines), before any stream is initialised: on, every
    // call takes each image's FastLineDetector segments (Segments: FLD's vector<Vec4f> as [m][4] floats, in its order, found on
    // fld_img: the grey image, or cvtColor(img, CV_RGB2GRAY) of a colour one, rectified where the handler remaps) beside its
    // images, through the overloads below, and runs fldKeyLines on them with lc.n_features; LSD does not run.  Where cfg has
    // no lines the segments are not read.
    using Segments = std::vector<float>;
    void useFLDLines(bool on) {
        session_.useFLDLines(on);
        fld_ = on;
    }
    // initialize(img_l[k], img_r[k], idx[k]) of stream ids[k], in one session call (idx optional)
    void initialize(const std::vector<int32_t>& ids, const std::vector<const uint8_t*>& img_l,
                    const std::vector<const uint8_t*>& img_r, const std::vector<int>& idx = {}) {
        initialize(ids, img_l, img_r, nullptr, nullptr, idx);
    }
    // the same on the FLD branch: seg_l[k] / seg_r[k] are the segments of img_l[k] / img_r[k]
    void initialize(const std::vector<int32_t>& ids, const std::vector<const uint8_t*>& img_l,
                    const std::vector<const uint8_t*>& img_r, const std::vector<Segments>& seg_l,
                    const std::vector<Segments>& seg_r, const std::vector<int>& idx = {}) {
        initialize(ids, img_l, img_r, &seg_l, &seg_r, idx);
    }
    // insertStereoPair(img_l[k], img_r[k], idx[k]) of stream ids[k]: f2fTracking of every named stream in one session call
    void insertStereoPairs(const std::vector<int32_t>& ids, const std::vector<const uint8_t*>& img_l,
                           const std::vector<const uint8_t*>& img_r, const std::vector<int>& idx = {}) {
        insertStereoPairs(ids, img_l, img_r, nullptr, nullptr, idx);
    }
    // the same on the FLD branch: seg_l[k] / seg_r[k] are the segments of img_l[k] / img_r[k]
    void insertStereoPairs(const std::vector<int32_t>& ids, const std::vector<const uint8_t*>& img_l,
                           const std::vector<const uint8_t*>& img_r, const std::vector<Segments>& seg_l,
                           const std::vector<Segments>& seg_r, const std::vector<int>& idx = {}) {
        insertStereoPairs(ids, img_l, img_r, &seg_l, &seg_r, idx);
    }
    // T frames per named stream in one session call (plstvo_stereo_session_run): img_l[t][k] / img_r[t][k] is stream ids[k]'s
    // frame of step t.  Each stream then stands as after T rounds of insertStereoPairs, optimizePose and updateFrame: its
    // prev_frame holds the last step's published pose, orb_fast_th the next frame's threshold, n_inliers* and n_stereo the
    // last step's, and per-frame calls can follow.  results (optional) receives [T][n] results.  The key-frame test is not
    // run here: the overload below runs it inside the call.  keepFeatures' arrays hold the last step.
    void insertStereoSequences(const std::vector<int32_t>& ids, const std::vector<std::vector<const uint8_t*>>& img_l,
                               const std::vector<std::vector<const uint8_t*>>& img_r, std::vector<PlPoseResult>* results = nullptr) {
        run(ids, img_l, img_r, nullptr, nullptr, results, nullptr, nullptr);
    }
    // the same on the FLD branch: seg_l[t][k] / seg_r[t][k] are the segments of img_l[t][k] / img_r[t][k]
    void insertStereoSequences(const std::vector<int32_t>& ids, const std::vector<std::vector<const uint8_t*>>& img_l,
                               const std::vector<std::vector<const uint8_t*>>& img_r,
                               const std::vector<std::vector<Segments>>& seg_l, const std::vector<std::vector<Segments>>& seg_r,
                               std::vector<PlPoseResult>* results = nullptr) {
        run(ids, img_l, img_r, &seg_l, &seg_r, results, nullptr, nullptr);
    }
    // A key frame of the key-frame overloads: stream id, step, and with keepFeatures its new stereo points and lines (pose
    // fields as published, Tfw before currFrameIsKF's reset)
    struct KeyFrame {
        int stream = 0, step = 0;
        StereoFrame frame;
    };
    // The same with the PL-SLAM test (plstvo_stereo_session_run_keyframes): per stream and step, needNewKF after optimizePose
    // and currFrameIsKF where it fires, from and back into each stream's kf.  A stream whose last step was a key frame has
    // prev_frame.Tfw = I and Tfw_cov = I, as currFrameIsKF leaves curr_frame.  Returns the [T][n] tests; results (optional)
    // receives [T][n] results, and keyframes (optional, with keepFeatures on) each key frame in (step, call position) order.
    std::vector<PlKeyframeResult> insertStereoSequences(const std::vector<int32_t>& ids,
                                                        const std::vector<std::vector<const uint8_t*>>& img_l,
                                                        const std::vector<std::vector<const uint8_t*>>& img_r,
                                                        std::vector<PlPoseResult>* results, std::vector<KeyFrame>* keyframes) {
        std::vector<PlKeyframeResult> kf;
        run(ids, img_l, img_r, nullptr, nullptr, results, &kf, keyframes);
        return kf;
    }
    // the same on the FLD branch, segments as in the plain FLD overload
    std::vector<PlKeyframeResult> insertStereoSequences(const std::vector<int32_t>& ids,
                                                        const std::vector<std::vector<const uint8_t*>>& img_l,
                                                        const std::vector<std::vector<const uint8_t*>>& img_r,
                                                        const std::vector<std::vector<Segments>>& seg_l,
                                                        const std::vector<std::vector<Segments>>& seg_r,
                                                        std::vector<PlPoseResult>* results, std::vector<KeyFrame>* keyframes) {
        std::vector<PlKeyframeResult> kf;
        run(ids, img_l, img_r, &seg_l, &seg_r, results, &kf, keyframes);
        return kf;
    }

    // Uneven streams in one session call (plstvo_stereo_session_run_schedule): schedule[t][k] is 0 when stream ids[k] has no
    // frame at step t, 1 for insertStereoPairs, 2 for initialize (at orb_fast_th, as initialize() above); img_l[t] / img_r[t]
    // hold step t's frames of its non-zero entries in ids order.  Each stream then stands as after the per-frame initialize /
    // insertStereoPairs + optimizePose (+ needNewKF / currFrameIsKF with kf) + updateFrame calls of its entries, and a
    // stream with no entry is untouched.  results (optional) receives [T][n] results (rows of non-insert entries zero);
    // kf non-null runs the key-frame test and receives its [T][n] tests.  keepFeatures' arrays hold the last step's last
    // group (its inserts, or its initialised frames).
    void insertStereoSequences(const std::vector<int32_t>& ids, const std::vector<std::vector<uint8_t>>& schedule,
                               const std::vector<std::vector<const uint8_t*>>& img_l,
                               const std::vector<std::vector<const uint8_t*>>& img_r,
                               std::vector<PlPoseResult>* results = nullptr, std::vector<PlKeyframeResult>* kf = nullptr) {
        runSchedule(ids, schedule, img_l, img_r, nullptr, nullptr, results, kf);
    }
    // the same on the FLD branch: seg_l[t][j] / seg_r[t][j] are the segments of img_l[t][j] / img_r[t][j]
    void insertStereoSequences(const std::vector<int32_t>& ids, const std::vector<std::vector<uint8_t>>& schedule,
                               const std::vector<std::vector<const uint8_t*>>& img_l,
                               const std::vector<std::vector<const uint8_t*>>& img_r,
                               const std::vector<std::vector<Segments>>& seg_l, const std::vector<std::vector<Segments>>& seg_r,
                               std::vector<PlPoseResult>* results = nullptr, std::vector<PlKeyframeResult>* kf = nullptr) {
        runSchedule(ids, schedule, img_l, img_r, &seg_l, &seg_r, results, kf);
    }

private:
    // the scheduled insertStereoSequences: the session call, then each stream's HandlerState as its last entry leaves it
    void runSchedule(const std::vector<int32_t>& ids, const std::vector<std::vector<uint8_t>>& schedule,
                     const std::vector<std::vector<const uint8_t*>>& img_l, const std::vector<std::vector<const uint8_t*>>& img_r,
                     const std::vector<std::vector<Segments>>* fl, const std::vector<std::vector<Segments>>* fr,
                     std::vector<PlPoseResult>* results, std::vector<PlKeyframeResult>* kf) {
        const char* who = "StereoStreamsHandler::insertStereoSequences";
        const size_t n = ids.size(), T = schedule.size();
        clearPlots(ids);
        if (img_l.size() != T || img_r.size() != T) throw Error(PLSTVO_E_INVALID, std::string(who) + ": one image list per step");
        std::vector<int32_t> th0, th_init;
        std::vector<PlPrior> priors;
        std::vector<PlKeyframeState> state;
        std::vector<uint8_t> flat;
        std::vector<const uint8_t*> l, r;
        std::vector<Segments> sl, sr;
        for (int32_t id : ids) {
            const Stream& s = at(id);
            th0.push_back(s.orb_fast_th);
            priors.push_back(priorOf(s.prev_frame));
            state.push_back(s.kf.state());
        }
        for (size_t t = 0; t < T; ++t) {
            if (schedule[t].size() != n) throw Error(PLSTVO_E_INVALID, std::string(who) + ": one schedule entry per stream and step");
            size_t m = 0;
            for (uint8_t c : schedule[t]) {
                flat.push_back(c);
                if (c) th_init.push_back(c == 2 ? hcfg_.orb_fast_th : 0);   // :38; an insert's threshold is the device's
                m += c != 0;
            }
            if (img_l[t].size() != m || img_r[t].size() != m)
                throw Error(PLSTVO_E_INVALID, std::string(who) + ": one image per non-zero entry");
            l.insert(l.end(), img_l[t].begin(), img_l[t].end());
            r.insert(r.end(), img_r[t].begin(), img_r[t].end());
            if (fl && fr) {
                if ((*fl)[t].size() != m || (*fr)[t].size() != m)
                    throw Error(PLSTVO_E_INVALID, std::string(who) + ": one segment list per image");
                sl.insert(sl.end(), (*fl)[t].begin(), (*fl)[t].end());
                sr.insert(sr.end(), (*fr)[t].begin(), (*fr)[t].end());
            }
        }
        if (fl && fr && (fl->size() != T || fr->size() != T))
            throw Error(PLSTVO_E_INVALID, std::string(who) + ": one segment list per image");
        if (T == 0 || n == 0 || l.empty()) return;
        pack_.pack(cam_.width, cam_.height, channels_, l, r, th_init, who);
        attachLines(fl ? &sl : nullptr, fr ? &sr : nullptr, who);
        std::vector<PlPoseResult> res(n * T);
        std::vector<int32_t> ns(4 * n * T);
        const PlKeyframeConfig kc = hcfg_.keyframes();
        if (kf) kf->assign(n * T, PlKeyframeResult{});
        session_.runSchedule(hcfg_.device(), kf ? &kc : nullptr, (int)n, ids.data(), (int)T, flat.data(), pack_.view, th0.data(),
                             priors.data(), kf ? state.data() : nullptr, res.data(), kf ? kf->data() : nullptr, nullptr,
                             ns.data());
        // the last step with entries: what keepFeatures reads, its insert group or else its initialize group
        size_t last = T;
        for (size_t t = T; t-- > 0 && last == T;)
            for (uint8_t c : schedule[t]) last = c ? t : last;
        std::vector<int32_t> read_ids, read_ns;
        bool read_insert = false;
        for (size_t k = 0; k < n; ++k) read_insert = read_insert || schedule[last][k] == 1;
        for (size_t k = 0; k < n; ++k) {
            const uint8_t c = schedule[last][k];
            if (c != (read_insert ? 1 : 2)) continue;
            read_ids.push_back(ids[k]);
            read_ns.insert(read_ns.end(), ns.begin() + 4 * (last * n + k) + (read_insert ? 0 : 2), ns.begin() + 4 * (last * n + k) + 4);
        }
        if (keep_) session_.read((int)read_ids.size(), read_ns.data(), read_insert, read_);
        // each stream's entries replayed in order on its HandlerState, as the per-frame calls leave it: initialize resets the
        // frame, threshold and key-frame test; an insert publishes its result (optimizePose), applies currFrameIsKF's pose
        // reset where the device's test fired, and updateFrame moves the frame into prev_frame with the next threshold
        for (size_t k = 0; k < n; ++k) {
            Stream& s = streams_[(size_t)ids[k]];
            size_t last_insert = T;
            bool insert_last = false;   // no initialize after the last insert
            for (size_t t = 0; t < T; ++t) {
                const uint8_t c = schedule[t][k];
                if (!c) continue;
                s.has_prev = true;
                insert_last = c == 1;
                if (c == 2) {   // as initialize() above
                    s.initialize(hcfg_, StereoFrame{});
                    s.curr_frame = StereoFrame{};
                    continue;
                }
                const PlPoseResult& r = res[t * n + k];
                s.result = r;
                std::copy(ns.begin() + 4 * (t * n + k), ns.begin() + 4 * (t * n + k) + 4, s.n_stereo.begin());
                s.curr_frame = StereoFrame{};
                s.optimizePose(r);
                if (kf && (*kf)[t * n + k].new_kf) {   // currFrameIsKF on curr_frame (the test's state: below)
                    s.curr_frame.Tfw = se3::identity4();
                    identityCov(s.curr_frame.Tfw_cov);
                }
                s.updateFrame(hcfg_);
                last_insert = t;
            }
            if (kf && insert_last) {   // the device's test as it stands after the stream's last insert
                s.kf = KeyframeTest::fromState(state[k]);
                const PlKeyframeResult& kl = (*kf)[last_insert * n + k];
                s.kf.entropy_curr = kl.entropy_curr;
                s.kf.entropy_ratio = kl.entropy_ratio;
                s.kf.kf_t = kl.t;
                s.kf.kf_r = kl.r;
            }
        }
        if (keep_) detail::splitRead(read_, read_ns.data(), read_insert ? 4 : 2, named(read_ids), &HandlerState::prev_frame);
        if (results) *results = std::move(res);
    }
    // the FLD branch's key lines of the packed frames (fl / fr null: none given)
    void attachLines(const std::vector<Segments>* fl, const std::vector<Segments>* fr, const char* who) {
        if (!fl != !fr) throw Error(PLSTVO_E_INVALID, std::string(who) + ": segments for both sides or neither");
        if (fl && !fld_) throw Error(PLSTVO_E_INVALID, std::string(who) + ": segments given: useFLDLines(true) first");
        if (!fl && fld_ && has_lines_)
            throw Error(PLSTVO_E_INVALID, std::string(who) + ": the FLD branch takes each image's segments");
        if (fl && has_lines_) pack_.addFLDLines(cam_.width, cam_.height, lsd_nfeatures_, *fl, *fr, who);
    }
    void initialize(const std::vector<int32_t>& ids, const std::vector<const uint8_t*>& img_l,
                    const std::vector<const uint8_t*>& img_r, const std::vector<Segments>* fl, const std::vector<Segments>* fr,
                    const std::vector<int>& idx) {
        const std::vector<int32_t> th(ids.size(), hcfg_.orb_fast_th);   // :38
        pack_.pack(cam_.width, cam_.height, channels_, img_l, img_r, th, "StereoStreamsHandler::initialize");
        attachLines(fl, fr, "StereoStreamsHandler::initialize");
        std::vector<int32_t> ns(2 * ids.size());
        session_.initialize((int)ids.size(), ids.data(), pack_.view, ns.data());
        if (keep_) session_.read((int)ids.size(), ns.data(), false, read_);
        for (size_t k = 0; k < ids.size(); ++k) {
            Stream& s = streams_[(size_t)ids[k]];
            StereoFrame frame;
            frame.frame_idx = k < idx.size() ? idx[k] : 0;
            s.initialize(hcfg_, std::move(frame));
            s.curr_frame = StereoFrame{};   // here only: the single handlers' initialize leaves curr_frame as it was
            s.has_prev = true;
        }
        if (keep_) detail::splitRead(read_, ns.data(), 2, named(ids), &HandlerState::prev_frame);
        splitPlot(ids);
    }
    void insertStereoPairs(const std::vector<int32_t>& ids, const std::vector<const uint8_t*>& img_l,
                           const std::vector<const uint8_t*>& img_r, const std::vector<Segments>* fl,
                           const std::vector<Segments>* fr, const std::vector<int>& idx) {
        std::vector<int32_t> th;
        std::vector<PlPrior> priors;
        for (int32_t id : ids) {
            const Stream& s = at(id);
            if (!s.has_prev) throw Error(PLSTVO_E_INVALID, "StereoStreamsHandler: initialize() the stream first");
            th.push_back(s.orb_fast_th);
            priors.push_back(priorOf(s.prev_frame));
        }
        pack_.pack(cam_.width, cam_.height, channels_, img_l, img_r, th, "StereoStreamsHandler::insertStereoPairs");
        attachLines(fl, fr, "StereoStreamsHandler::insertStereoPairs");
        std::vector<PlPoseResult> res(ids.size());
        std::vector<int32_t> ns(4 * ids.size());
        session_.insert((int)ids.size(), ids.data(), pack_.view, priors.data(), res.data(), ns.data());
        if (keep_) session_.read((int)ids.size(), ns.data(), true, read_);
        for (size_t k = 0; k < ids.size(); ++k) {
            Stream& s = streams_[(size_t)ids[k]];
            s.curr_frame = StereoFrame{};
            s.curr_frame.frame_idx = k < idx.size() ? idx[k] : 0;
            s.result = res[k];
            std::copy(ns.begin() + 4 * k, ns.begin() + 4 * k + 4, s.n_stereo.begin());
            s.tracked(s.result);
        }
        if (keep_) detail::splitRead(read_, ns.data(), 4, named(ids), &HandlerState::curr_frame);
        splitPlot(ids);
    }
    // a run draws nothing: the streams it names lose their last image
    void clearPlots(const std::vector<int32_t>& ids) {
        for (int32_t id : ids)
            if (id >= 0 && (size_t)id < streams_.size()) streams_[(size_t)id].plot.clear();
    }
    // plotFrames: the last call's images into the named streams' plot, in call order
    void splitPlot(const std::vector<int32_t>& ids) {
        if (!plot_) return;
        const size_t px = (size_t)cam_.width * cam_.height * 3;
        session_.readPlot((int)ids.size(), cam_.width, cam_.height, plot_read_);
        for (size_t k = 0; k < ids.size(); ++k)
            streams_[(size_t)ids[k]].plot.assign(plot_read_.begin() + k * px, plot_read_.begin() + (k + 1) * px);
    }

public:
    void optimizePose(int id) { Stream& s = at(id); s.optimizePose(s.result); }
    void updateFrame(int id) { at(id).updateFrame(hcfg_); }
    bool needNewKF(int id) { return at(id).needNewKF(hcfg_); }
    void currFrameIsKF(int id) { at(id).currFrameIsKF(); }

    // StereoImageHandler::keepFeatures for every stream: initialize fills the named streams' prev_frame arrays,
    // insertStereoPairs their curr_frame arrays and matches_pt / _ls, inlier_pt / _ls
    void keepFeatures(bool on) {
        session_.retain(on || plot_);   // plotting draws the retained rows
        keep_ = on;
    }
    // StereoImageHandler::plotFrames for every stream: initialize and insertStereoPairs fill the named streams' images; the
    // insertStereoSequences overloads draw nothing and clear the images of the streams they name
    void plotFrames(bool on) {
        if (on) session_.retain(true);
        session_.plot(on);
        if (!on && !keep_) session_.retain(false);
        plot_ = on;
        for (Stream& s : streams_) s.plot.clear();
    }
    // StereoImageHandler::plotStereoFrame() of stream id: the image of the frame its last initialize / insertStereoPairs
    // produced ([height][width][3] BGR bytes; empty with plotFrames off, or after an insertStereoSequences naming it)
    const std::vector<uint8_t>& plotStereoFrame(int id) { return at(id).plot; }
    Stream& stream(int id) { return at(id); }
    int streams() const { return (int)streams_.size(); }
    const StereoSession& session() const { return session_; }

private:
    // the insertStereoSequences: kf null runs plstvo_stereo_session_run, else plstvo_stereo_session_run_keyframes; fl / fr
    // (FLD branch) [T][n] segments
    void run(const std::vector<int32_t>& ids, const std::vector<std::vector<const uint8_t*>>& img_l,
             const std::vector<std::vector<const uint8_t*>>& img_r, const std::vector<std::vector<Segments>>* fl,
             const std::vector<std::vector<Segments>>* fr, std::vector<PlPoseResult>* results,
             std::vector<PlKeyframeResult>* kf, std::vector<KeyFrame>* keyframes) {
        const size_t n = ids.size(), T = img_l.size();
        clearPlots(ids);
        if (img_r.size() != T) throw Error(PLSTVO_E_INVALID, "StereoStreamsHandler::insertStereoSequences: T differs between sides");
        std::vector<int32_t> th0;
        std::vector<PlPrior> priors;
        std::vector<PlKeyframeState> state;
        std::vector<const uint8_t*> l, r;
        for (int32_t id : ids) {
            const Stream& s = at(id);
            if (!s.has_prev) throw Error(PLSTVO_E_INVALID, "StereoStreamsHandler: initialize() the stream first");
            th0.push_back(s.orb_fast_th);
            priors.push_back(priorOf(s.prev_frame));
            state.push_back(s.kf.state());
        }
        if (kf) kf->clear();
        if (keyframes) keyframes->clear();
        for (size_t t = 0; t < T; ++t) {
            if (img_l[t].size() != n || img_r[t].size() != n)
                throw Error(PLSTVO_E_INVALID, "StereoStreamsHandler::insertStereoSequences: one image per stream and step");
            l.insert(l.end(), img_l[t].begin(), img_l[t].end());
            r.insert(r.end(), img_r[t].begin(), img_r[t].end());
        }
        if (T == 0 || n == 0) return;
        pack_.pack(cam_.width, cam_.height, channels_, l, r, std::vector<int32_t>(n * T, 0),
                   "StereoStreamsHandler::insertStereoSequences");
        std::vector<Segments> sl, sr;   // step-major, as the images
        if (fl && fr) {
            if (fl->size() != T || fr->size() != T)
                throw Error(PLSTVO_E_INVALID, "StereoStreamsHandler::insertStereoSequences: one segment list per image");
            for (size_t t = 0; t < T; ++t) {
                sl.insert(sl.end(), (*fl)[t].begin(), (*fl)[t].end());
                sr.insert(sr.end(), (*fr)[t].begin(), (*fr)[t].end());
            }
        }
        attachLines(fl ? &sl : nullptr, fr ? &sr : nullptr, "StereoStreamsHandler::insertStereoSequences");
        PlStereoImages frames = pack_.view;
        frames.fast_th = nullptr;
        std::vector<PlPoseResult> res(n * T);
        std::vector<int32_t> th((T + 1) * n), ns(4 * n * T);
        // th0 of 0 would mean the session's configured threshold, which the handler's ORB config sets to 0 as well
        if (kf) {
            kf->resize(n * T);
            session_.runKeyframes(hcfg_.device(), hcfg_.keyframes(), (int)n, ids.data(), (int)T, frames, th0.data(),
                                  priors.data(), state.data(), res.data(), kf->data(), th.data(), ns.data());
            if (keyframes && keep_) {
                std::vector<int32_t> rows;
                session_.readKeyframes(read_, rows);
                detail::ReadCursor c{read_};
                for (size_t j = 0; j < rows.size() / 4; ++j) {
                    KeyFrame f;
                    f.step = rows[4 * j];
                    f.stream = rows[4 * j + 1];
                    c.frameFromRead((size_t)rows[4 * j + 2], (size_t)rows[4 * j + 3], f.frame);
                    size_t k = 0;
                    while (ids[k] != f.stream) ++k;
                    publishPose(res[(size_t)f.step * n + k], f.frame);
                    keyframes->push_back(std::move(f));
                }
            }
        } else {
            session_.run(hcfg_.device(), (int)n, ids.data(), (int)T, frames, th0.data(), priors.data(), res.data(), th.data(),
                         ns.data());
        }
        const int32_t* ns_last = ns.data() + 4 * n * (T - 1);
        if (keep_) session_.read((int)n, ns_last, true, read_);
        for (size_t k = 0; k < n; ++k) {
            Stream& s = streams_[(size_t)ids[k]];
            const PlPoseResult& last = res[(T - 1) * n + k];
            s.result = last;
            std::copy(ns_last + 4 * k, ns_last + 4 * k + 4, s.n_stereo.begin());
            // the last step's optimizePose (so n_inliers* are its inlier counts, not f2fTracking's matched counts) and
            // updateFrame, with the threshold the device carried
            s.curr_frame = StereoFrame{};
            s.optimizePose(last);
            s.prev_frame = std::move(s.curr_frame);
            s.curr_frame = StereoFrame{};
            s.orb_fast_th = th[T * n + k];
            if (kf) {
                s.kf = KeyframeTest::fromState(state[k]);
                const PlKeyframeResult& kl = (*kf)[(T - 1) * n + k];
                s.kf.entropy_curr = kl.entropy_curr;
                s.kf.entropy_ratio = kl.entropy_ratio;
                s.kf.kf_t = kl.t;
                s.kf.kf_r = kl.r;
                if (kl.new_kf) {   // currFrameIsKF on the frame that became prev_frame: its Tfw / Tfw_cov (kf is the device's)
                    s.prev_frame.Tfw = se3::identity4();
                    identityCov(s.prev_frame.Tfw_cov);
                }
            }
        }
        if (keep_) detail::splitRead(read_, ns_last, 4, named(ids), &HandlerState::prev_frame);
        if (results) *results = std::move(res);
    }
    Stream& at(int id) {
        if (id < 0 || id >= (int)streams_.size()) throw Error(PLSTVO_E_INVALID, "StereoStreamsHandler: stream id out of range");
        return streams_[(size_t)id];
    }
    // the streams ids name, in call order
    std::vector<HandlerState*> named(const std::vector<int32_t>& ids) {
        std::vector<HandlerState*> s;
        for (int32_t id : ids) s.push_back(&at(id));
        return s;
    }
    PlCamera cam_;
    HandlerConfig hcfg_;
    StereoSession session_;
    std::vector<Stream> streams_;
    int channels_ = 1;   // bytes per pixel of the images: the rectifier's channels
    int lsd_nfeatures_ = 0;   // lsd_nfeatures, the FLD branch's truncation
    bool has_lines_ = true;
    bool fld_ = false;        // useFLDLines
    detail::StereoImagesBatch pack_;
    bool keep_ = false;
    StereoSession::Frames read_;
    bool plot_ = false;
    std::vector<uint8_t> plot_read_;
};

}  // namespace plstvo
