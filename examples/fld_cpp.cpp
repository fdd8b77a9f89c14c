// C++ host example: the reference's FLD line branch (use_fld_lines) on a stereo session.  The caller detects each image's
// line segments and plstvo::fldKeyLines turns them into key lines as detectLineFeatures' FLD branch does; the session then
// takes those key lines instead of running LSD.  This repository does not link cv::ximgproc, so plstvo::detectLSD's
// segments stand in for FastLineDetector::detect's output.  LSD's key lines are already clamped, filtered and truncated, so
// the FLD session must then equal a plain LSD session: the example initialises both on the same synthetic frames and inserts
// T frames per stream.  It then does the same with two plstvo::StereoStreamsHandlers, the FLD one fed each image's
// segments beside the images: initialize, per-frame insertStereoPairs / optimizePose / updateFrame, and both
// insertStereoSequences (plain, and with the key-frame test).  Prints the poses and exits 0 when every result, threshold and
// key-frame decision is the same byte for byte, 1 otherwise.
//   g++ -std=c++17 -Iinclude examples/fld_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o fld_cpp
#include <cstdio>
#include <cstring>

#include "plstvo.hpp"

namespace {
constexpr int W = 320, H = 240, S = 3, T = 3, DISP = 12;

// a texture of random grey rectangles, 64 px wider and taller than the views (a linear congruential generator)
std::vector<uint8_t> texture(uint32_t seed) {
    const int tw = W + DISP + 64, th = H + 64;
    std::vector<uint8_t> t((size_t)tw * th, 128);
    auto next = [&seed]() { return seed = seed * 1664525u + 1013904223u; };
    for (int r = 0; r < 900; ++r) {
        const int x = (int)(next() % (uint32_t)tw), y = (int)(next() % (uint32_t)th);
        const int w = 2 + (int)(next() % 24u), h = 2 + (int)(next() % 24u);
        const uint8_t v = (uint8_t)(next() >> 24);
        for (int yy = y; yy < std::min(y + h, th); ++yy)
            for (int xx = x; xx < std::min(x + w, tw); ++xx) t[(size_t)yy * tw + xx] = v;
    }
    return t;
}

std::vector<uint8_t> view(const std::vector<uint8_t>& tex, int x0, int y0) {
    const int tw = W + DISP + 64;
    std::vector<uint8_t> v((size_t)W * H);
    for (int y = 0; y < H; ++y) std::memcpy(&v[(size_t)y * W], &tex[(size_t)(y + y0) * tw + x0], W);
    return v;
}
}  // namespace

int main() {
    PlCamera cam{300.0, 300.0, 160.0, 120.0, 0.2, W, H};
    PlConfig cfg;
    plstvo_kitti_config(&cfg);
    PlStereoMatchConfig mc;
    plstvo_default_stereo_match_config(&mc);
    PlStereoConfig sc;
    plstvo_default_stereo_config(&sc);
    PlOrbDetectConfig oc;
    plstvo_default_orb_detect_config(&oc);
    oc.n_features = 500;
    PlLsdConfig lc;
    plstvo_default_lsd_config(&lc);
    plstvo::Context ctx;
    plstvo::StereoSession lsd(ctx, cam, cfg, mc, sc, oc, lc, S), fld(ctx, cam, cfg, mc, sc, oc, lc, S);
    fld.useFLDLines(true);
    std::vector<std::vector<uint8_t>> tex;
    for (int s = 0; s < S; ++s) tex.push_back(texture(4321u + 31u * (uint32_t)s));
    const std::vector<int32_t> ids = {1, 2, 0};
    bool same = true;
    for (int f = 0; f <= T; ++f) {
        std::vector<std::vector<uint8_t>> img_l, img_r;
        std::vector<plstvo::StereoImageFrame> frames(ids.size());
        for (size_t k = 0; k < ids.size(); ++k) {
            const int x0 = 2 + f * (2 + ids[k]), y0 = 1 + f;
            img_l.push_back(view(tex[(size_t)ids[k]], x0, y0));
            img_r.push_back(view(tex[(size_t)ids[k]], x0 + DISP, y0));
        }
        for (size_t k = 0; k < ids.size(); ++k) {
            plstvo::StereoImageFrame& fr = frames[k];
            fr.img_l = img_l[k].data();
            fr.img_r = img_r[k].data();
            for (int side = 0; side < 2; ++side) {   // the stand-in for fld->detect(fld_img, fld_lines), then the KeyLine step
                plstvo::KeyLines detected, kl;
                std::vector<int32_t> npix;
                plstvo::detectLSD(ctx, lc, side ? fr.img_r : fr.img_l, W, H, detected, npix);
                plstvo::fldKeyLines(W, H, lc.n_features, detected.seg, kl, npix);
                (side ? fr.seg_r : fr.seg_l) = kl.seg;
                (side ? fr.angle_r : fr.angle_l) = kl.angle;
                (side ? fr.npix_r : fr.npix_l) = npix;
            }
        }
        plstvo::detail::StereoImagesPack with_lines, images_only;
        plstvo::detail::packStereoImages(frames, W, H, with_lines);
        plstvo::detail::packStereoImages(frames, W, H, images_only);
        for (plstvo::StereoImageFrame& fr : frames) fr.seg_l = fr.seg_r = fr.angle_l = fr.angle_r = {}, fr.npix_l = fr.npix_r = {};
        plstvo::detail::dropLines(frames, images_only, "fld_cpp");
        const int n = (int)ids.size();
        if (f == 0) {
            lsd.initialize(n, ids.data(), images_only.view);
            fld.initialize(n, ids.data(), with_lines.view);
            continue;
        }
        std::vector<PlPoseResult> ra((size_t)n), rb((size_t)n);
        lsd.insert(n, ids.data(), images_only.view, nullptr, ra.data());
        fld.insert(n, ids.data(), with_lines.view, nullptr, rb.data());
        for (int k = 0; k < n; ++k) {
            same = same && std::memcmp(&ra[(size_t)k], &rb[(size_t)k], sizeof(PlPoseResult)) == 0;
            std::printf("stream %d frame %d good %d n_inliers_ls %d err_norm %.17g\n", ids[(size_t)k], f, rb[(size_t)k].good,
                        rb[(size_t)k].n_inliers_ls, rb[(size_t)k].err_norm);
        }
    }
    std::printf(same ? "the FLD session equals the LSD session\n" : "the FLD session differs from the LSD session\n");

    // ---- the handler surface ----
    plstvo::HandlerConfig hc;
    hc.fast_feat_th = 20;
    hc.max_kf_t_dist = 0.01;   // the key-frame test fires on some steps
    plstvo::StereoStreamsHandler hl(ctx, cam, cfg, mc, sc, oc, lc, S, hc), hf(ctx, cam, cfg, mc, sc, oc, lc, S, hc);
    hf.useFLDLines(true);
    using Seg = plstvo::StereoStreamsHandler::Segments;
    auto segments = [&](const uint8_t* img) {   // the stand-in for fld->detect(fld_img, fld_lines)
        plstvo::KeyLines kl;
        std::vector<int32_t> npix;
        plstvo::detectLSD(ctx, lc, img, W, H, kl, npix);
        return Seg(kl.seg);
    };
    std::vector<std::vector<std::vector<uint8_t>>> views_l(S), views_r(S);   // [stream][frame]
    const int NF = 7;
    for (int s = 0; s < S; ++s)
        for (int f = 0; f < NF; ++f) {
            const int x0 = 2 + f * (2 + s), y0 = 1 + f;
            views_l[(size_t)s].push_back(view(tex[(size_t)s], x0, y0));
            views_r[(size_t)s].push_back(view(tex[(size_t)s], x0 + DISP, y0));
        }
    auto images = [&](int f, bool left) {
        std::vector<const uint8_t*> v;
        for (int32_t id : ids) v.push_back((left ? views_l : views_r)[(size_t)id][(size_t)f].data());
        return v;
    };
    auto segs = [&](int f, bool left) {
        std::vector<Seg> v;
        for (const uint8_t* img : images(f, left)) v.push_back(segments(img));
        return v;
    };
    auto same_streams = [&]() {
        bool ok = true;
        for (int32_t id : ids) {
            const plstvo::StereoStreamsHandler::Stream &a = hl.stream(id), &b = hf.stream(id);
            ok = ok && std::memcmp(&a.result, &b.result, sizeof(PlPoseResult)) == 0 && a.orb_fast_th == b.orb_fast_th &&
                 a.n_stereo == b.n_stereo && a.prev_frame.Tfw == b.prev_frame.Tfw && a.prev_frame.Tfw_cov == b.prev_frame.Tfw_cov;
        }
        return ok;
    };
    hl.initialize(ids, images(0, true), images(0, false));
    hf.initialize(ids, images(0, true), images(0, false), segs(0, true), segs(0, false));
    bool handlers = true;
    for (int f = 1; f <= 2; ++f) {   // the reference's loop, frame by frame
        hl.insertStereoPairs(ids, images(f, true), images(f, false));
        hf.insertStereoPairs(ids, images(f, true), images(f, false), segs(f, true), segs(f, false));
        for (int32_t id : ids) {
            hl.optimizePose(id);
            hf.optimizePose(id);
            hl.updateFrame(id);
            hf.updateFrame(id);
            std::printf("handler stream %d frame %d th %d err_norm %.17g\n", id, f, hf.stream(id).orb_fast_th,
                        hf.stream(id).result.err_norm);
        }
        handlers = handlers && same_streams();
    }
    std::vector<std::vector<const uint8_t*>> sl, sr;   // frames 3, 4 in one call, then 5, 6 with the key-frame test
    std::vector<std::vector<Seg>> gl, gr;
    for (int f = 3; f <= 4; ++f) {
        sl.push_back(images(f, true));
        sr.push_back(images(f, false));
        gl.push_back(segs(f, true));
        gr.push_back(segs(f, false));
    }
    std::vector<PlPoseResult> ra, rb;
    hl.insertStereoSequences(ids, sl, sr, &ra);
    hf.insertStereoSequences(ids, sl, sr, gl, gr, &rb);
    handlers = handlers && ra.size() == rb.size() && std::memcmp(ra.data(), rb.data(), ra.size() * sizeof(PlPoseResult)) == 0 &&
               same_streams();
    for (int f = 5; f <= 6; ++f) {
        sl[(size_t)f - 5] = images(f, true);
        sr[(size_t)f - 5] = images(f, false);
        gl[(size_t)f - 5] = segs(f, true);
        gr[(size_t)f - 5] = segs(f, false);
    }
    const std::vector<PlKeyframeResult> ka = hl.insertStereoSequences(ids, sl, sr, &ra, nullptr);
    const std::vector<PlKeyframeResult> kb = hf.insertStereoSequences(ids, sl, sr, gl, gr, &rb, nullptr);
    int n_kf = 0;
    for (size_t j = 0; j < ka.size() && j < kb.size(); ++j) {
        handlers = handlers && ka[j].new_kf == kb[j].new_kf && ka[j].N_prevKF_currF == kb[j].N_prevKF_currF;
        n_kf += kb[j].new_kf;
    }
    handlers = handlers && ka.size() == kb.size() && std::memcmp(ra.data(), rb.data(), ra.size() * sizeof(PlPoseResult)) == 0 &&
               same_streams();
    std::printf("handler key frames %d\n", n_kf);
    std::printf(handlers ? "the FLD handler equals the LSD handler\n" : "the FLD handler differs from the LSD handler\n");
    return same && handlers ? 0 : 1;
}
