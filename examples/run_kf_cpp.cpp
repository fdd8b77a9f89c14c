// C++ host example: a PL-SLAM front end's frame loop (app/imagesStVO.cpp:88-124 with needNewKF / currFrameIsKF) over several
// streams and several frames in one call.  Two plstvo::StereoStreamsHandlers over the same frames, both keeping features:
// one runs T frames per stream with the key-frame overload of insertStereoSequences (plstvo_stereo_session_run_keyframes:
// the test runs on the device, and each key frame's stereo features come back), the other the per-frame loop of
// insertStereoPairs, optimizePose, needNewKF, currFrameIsKF and updateFrame.  The frames are run_cpp.cpp's synthetic views.
// Prints every test and exits 0 when the two agree: results byte for byte, the decisions and counters, each key frame's
// points and lines, each stream's key-frame state, and a further per-frame insert; 1 otherwise.
//   g++ -std=c++17 -Iinclude examples/run_kf_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o run_kf_cpp
#include <cstdio>
#include <cstring>

#include "plstvo.hpp"

namespace {
constexpr int W = 320, H = 240, S = 4, T = 6, DISP = 12;

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
    hc.max_kf_t_dist = 0.02;   // the views move a few pixels per frame: a short baseline makes key frames every few frames
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
    run.keepFeatures(true);
    loop.keepFeatures(true);
    run.initialize(ids, frame(0, true), frame(0, false));
    loop.initialize(ids, frame(0, true), frame(0, false));
    std::vector<std::vector<const uint8_t*>> seq_l, seq_r;
    for (int t = 1; t <= T; ++t) {
        seq_l.push_back(frame(t, true));
        seq_r.push_back(frame(t, false));
    }
    std::vector<PlPoseResult> res;
    std::vector<plstvo::StereoStreamsHandler::KeyFrame> kfs;
    const std::vector<PlKeyframeResult> kf = run.insertStereoSequences(ids, seq_l, seq_r, &res, &kfs);
    bool same = res.size() == (size_t)T * ids.size() && kf.size() == res.size();
    size_t next_kf = 0;
    for (int t = 1; t <= T; ++t) {
        loop.insertStereoPairs(ids, frame(t, true), frame(t, false));
        for (size_t k = 0; k < ids.size(); ++k) {
            const int id = ids[k];
            loop.optimizePose(id);
            const size_t row = (size_t)(t - 1) * ids.size() + k;
            const PlPoseResult& r = loop.stream(id).result;
            same = same && std::memcmp(&r, &res[row], sizeof r) == 0;
            const bool is_kf = loop.needNewKF(id);
            same = same && (int)is_kf == kf[row].new_kf && loop.stream(id).kf.N_prevKF_currF == kf[row].N_prevKF_currF;
            std::printf("stream %d step %d key frame %d (%d) N %d t %.6f r %.6f ratio %.6f\n", id, t, (int)is_kf,
                        kf[row].new_kf, kf[row].N_prevKF_currF, kf[row].t, kf[row].r, kf[row].entropy_ratio);
            if (is_kf) {
                const plstvo::StereoFrame& f = loop.stream(id).curr_frame;
                const bool found = next_kf < kfs.size() && kfs[next_kf].stream == id && kfs[next_kf].step == t - 1;
                same = same && found && kfs[next_kf].frame.pt_P == f.pt_P && kfs[next_kf].frame.pdesc == f.pdesc &&
                       kfs[next_kf].frame.ls_sP == f.ls_sP && kfs[next_kf].frame.ldesc == f.ldesc;
                ++next_kf;
                loop.currFrameIsKF(id);
            }
            loop.updateFrame(id);
        }
    }
    same = same && next_kf == kfs.size();
    for (int32_t id : ids) {
        const plstvo::StereoStreamsHandler::Stream &a = run.stream(id), &b = loop.stream(id);
        same = same && a.orb_fast_th == b.orb_fast_th && a.prev_frame.Tfw == b.prev_frame.Tfw &&
               a.prev_frame.Tfw_cov == b.prev_frame.Tfw_cov && a.kf.N_prevKF_currF == b.kf.N_prevKF_currF &&
               a.kf.prev_f_iskf == b.kf.prev_f_iskf && a.kf.T_prevKF == b.kf.T_prevKF &&
               a.kf.entropy_first_prevKF == b.kf.entropy_first_prevKF;
    }
    // per-frame calls follow the run seamlessly
    run.insertStereoPairs(ids, frame(T + 1, true), frame(T + 1, false));
    loop.insertStereoPairs(ids, frame(T + 1, true), frame(T + 1, false));
    for (int32_t id : ids) same = same && std::memcmp(&run.stream(id).result, &loop.stream(id).result, sizeof(PlPoseResult)) == 0;
    std::printf("%zu key frames\n", kfs.size());
    std::printf(same ? "run with key frames equals the per-frame loop\n" : "run with key frames differs from the per-frame loop\n");
    return same ? 0 : 1;
}
