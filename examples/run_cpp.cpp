// C++ host example: the reference's frame loop (app/imagesStVO.cpp:88-124) over several streams and several frames in one
// call.  Two plstvo::StereoStreamsHandlers over the same frames: one runs T frames per stream with insertStereoSequences
// (plstvo_stereo_session_run: the adaptive FAST threshold and the prior carried on the device), the other the per-frame
// loop of insertStereoPairs, optimizePose and updateFrame.  The frames are synthetic: each stream views its own random
// texture from a window that moves by a few pixels per frame, the right view shifted by a fixed disparity.  Prints each
// stream's thresholds and poses and exits 0 when the two agree byte for byte (every step's results, then the state a
// further per-frame insert starts from), 1 otherwise.
//   g++ -std=c++17 -Iinclude examples/run_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o run_cpp
#include <cstdio>
#include <cstring>

#include "plstvo.hpp"

namespace {
constexpr int W = 320, H = 240, S = 4, T = 5, DISP = 12;

// a texture of random grey rectangles, 64 px wider and taller than the views (a linear congruential generator: no library
// randomness, the same bytes everywhere)
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
    mc.min_ratio_12_p = 0.75;
    PlStereoConfig sc;
    plstvo_default_stereo_config(&sc);
    PlOrbDetectConfig oc;
    plstvo_default_orb_detect_config(&oc);
    oc.n_features = 500;
    PlLsdConfig lc;
    plstvo_default_lsd_config(&lc);
    plstvo::HandlerConfig hc;
    hc.fast_feat_th = 20;
    // frames [stream][frame]: frame 0 initialises, frames 1 .. T are the run
    std::vector<std::vector<std::vector<uint8_t>>> left(S), right(S);
    for (int s = 0; s < S; ++s) {
        const std::vector<uint8_t> tex = texture(1234u + 77u * (uint32_t)s);
        for (int f = 0; f <= T + 1; ++f) {
            const int x0 = 2 + f * (2 + s), y0 = 1 + f;
            left[(size_t)s].push_back(view(tex, x0, y0));
            right[(size_t)s].push_back(view(tex, x0 + DISP, y0));
        }
    }
    const std::vector<int32_t> ids = {2, 0, 3, 1};
    auto frame = [&](int f, bool l) {
        std::vector<const uint8_t*> v;
        for (int32_t id : ids) v.push_back((l ? left : right)[(size_t)id][(size_t)f].data());
        return v;
    };
    plstvo::Context ctx;
    plstvo::StereoStreamsHandler run(ctx, cam, cfg, mc, sc, oc, lc, S, hc), loop(ctx, cam, cfg, mc, sc, oc, lc, S, hc);
    run.initialize(ids, frame(0, true), frame(0, false));
    loop.initialize(ids, frame(0, true), frame(0, false));
    std::vector<std::vector<const uint8_t*>> seq_l, seq_r;
    for (int t = 1; t <= T; ++t) {
        seq_l.push_back(frame(t, true));
        seq_r.push_back(frame(t, false));
    }
    std::vector<PlPoseResult> res;
    run.insertStereoSequences(ids, seq_l, seq_r, &res);
    bool same = res.size() == (size_t)T * ids.size();
    for (int t = 1; t <= T; ++t) {
        loop.insertStereoPairs(ids, frame(t, true), frame(t, false));
        for (size_t k = 0; k < ids.size(); ++k) {
            const int id = ids[k];
            const int th = loop.stream(id).orb_fast_th;
            loop.optimizePose(id);
            const PlPoseResult& r = loop.stream(id).result;
            same = same && std::memcmp(&r, &res[(size_t)(t - 1) * ids.size() + k], sizeof r) == 0;
            loop.updateFrame(id);
            std::printf("stream %d step %d th %d good %d n_inliers_pt %d err_norm %.17g\n", id, t, th, r.good, r.n_inliers_pt,
                        r.err_norm);
        }
    }
    for (int32_t id : ids) {
        const plstvo::StereoStreamsHandler::Stream &a = run.stream(id), &b = loop.stream(id);
        same = same && a.orb_fast_th == b.orb_fast_th && a.prev_frame.DT == b.prev_frame.DT && a.prev_frame.Tfw == b.prev_frame.Tfw &&
               a.prev_frame.Tfw_cov == b.prev_frame.Tfw_cov && a.prev_frame.err_norm == b.prev_frame.err_norm &&
               a.n_stereo == b.n_stereo && a.n_inliers_pt == b.n_inliers_pt;
        std::printf("stream %d next th %d %d\n", id, a.orb_fast_th, b.orb_fast_th);
    }
    // per-frame calls follow the run seamlessly
    run.insertStereoPairs(ids, frame(T + 1, true), frame(T + 1, false));
    loop.insertStereoPairs(ids, frame(T + 1, true), frame(T + 1, false));
    for (int32_t id : ids) same = same && std::memcmp(&run.stream(id).result, &loop.stream(id).result, sizeof(PlPoseResult)) == 0;
    std::printf(same ? "run equals the per-frame loop\n" : "run differs from the per-frame loop\n");
    return same ? 0 : 1;
}
