// C++ host example: many stereo cameras whose frames arrive unevenly, all tracked in ONE plstvo::StereoStreamsHandler call
// (insertStereoSequences with a schedule: plstvo_stereo_session_run_schedule).  Each round is one step of the schedule: a
// camera with no frame that round idles (its kept frame, FAST threshold, prior and key-frame state carried), a camera seen
// for the first time (a late camera) or named for re-initialisation is initialised, and every other named camera is tracked
// (insertStereoPair, optimizePose, the key-frame test, updateFrame, as app/imagesStVO.cpp:88-124 per camera).  Every image
// goes up, is detected and described once for the whole call.  With "per-frame" the same log goes through the handler round
// by round instead (initialize, insertStereoPairs, optimizePose, needNewKF / currFrameIsKF, updateFrame), which prints the
// same; "no-kf" leaves the key-frame test out.  Reads one binary file: width, height, streams and rounds (int32), then per
// round the number of frames m (int32) and m times a stream id (int32; -(id + 1) re-initialises stream id) followed by its
// left and right grey images (width * height bytes each).  KITTI camera and config, the default ORB (1200 features, 4
// levels) and LSD options, min_ratio_12_p 0.75, the default HandlerConfig.  Prints, per tracked frame, the round, the
// stream, good, DT, Tfw and the key-frame decision, then each stream's handler state: its next FAST threshold, its last
// insert's inlier and stereo feature counts and err_norm, prev_frame's Tfw, Tfw_cov, DT, DT_cov and err_norm, and the
// key-frame test's state.
//   g++ -std=c++17 -Iinclude examples/schedule_cpp.cpp -Lstvo_pl_b200/lib -lplstvo_b200 -o schedule_cpp
#include <cstdio>
#include <fstream>
#include <string>

#include "plstvo.hpp"

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: schedule_cpp <file> [per-frame] [no-kf]\n"); return 2; }
    bool per_frame = false, keyframes = true;
    for (int i = 2; i < argc; ++i) {
        const std::string a = argv[i];
        if (a == "per-frame") per_frame = true;
        else if (a == "no-kf") keyframes = false;
        else { std::fprintf(stderr, "unknown option %s\n", argv[i]); return 2; }
    }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) return 2;
    int32_t hdr[4];
    f.read(reinterpret_cast<char*>(hdr), 16);
    if (!f || hdr[0] < 1 || hdr[1] < 1 || hdr[2] < 1 || hdr[3] < 0) return 2;
    const size_t px = (size_t)hdr[0] * hdr[1];
    const int S = hdr[2], T = hdr[3];
    PlCamera cam{};
    cam.fx = cam.fy = 718.856; cam.cx = 607.1928; cam.cy = 185.2157; cam.b = 0.537165719; cam.width = hdr[0]; cam.height = hdr[1];
    PlConfig cfg;
    plstvo_kitti_config(&cfg);
    PlStereoMatchConfig mc;
    plstvo_default_stereo_match_config(&mc);
    mc.min_ratio_12_p = 0.75;
    PlStereoConfig sc;
    plstvo_default_stereo_config(&sc);
    PlOrbDetectConfig oc;
    plstvo_default_orb_detect_config(&oc);
    PlLsdConfig lc;
    plstvo_default_lsd_config(&lc);
    std::vector<int32_t> ids;
    for (int id = 0; id < S; ++id) ids.push_back(id);
    // the schedule [T][S] and each step's images of its named cameras, in stream order
    std::vector<std::vector<uint8_t>> schedule((size_t)T, std::vector<uint8_t>((size_t)S, 0));
    std::vector<std::vector<const uint8_t*>> img_l((size_t)T), img_r((size_t)T);
    std::vector<std::vector<uint8_t>> store;
    std::vector<uint8_t> seen((size_t)S, 0);
    for (int t = 0; t < T; ++t) {
        int32_t m = 0;
        f.read(reinterpret_cast<char*>(&m), 4);
        if (!f || m < 0) return 2;
        std::vector<const uint8_t*> by_l((size_t)S, nullptr), by_r((size_t)S, nullptr);
        for (int k = 0; k < m; ++k) {
            int32_t id = -1;
            f.read(reinterpret_cast<char*>(&id), 4);
            const bool reinit = id < 0;
            if (reinit) id = -id - 1;
            if (!f || id >= S || schedule[(size_t)t][(size_t)id]) return 2;
            for (int side = 0; side < 2; ++side) {
                store.emplace_back(px);
                f.read(reinterpret_cast<char*>(store.back().data()), (std::streamsize)px);
            }
            if (!f) return 2;
            schedule[(size_t)t][(size_t)id] = reinit || !seen[(size_t)id] ? 2 : 1;
            seen[(size_t)id] = 1;
            by_l[(size_t)id] = store[store.size() - 2].data();
            by_r[(size_t)id] = store.back().data();
        }
        for (int id = 0; id < S; ++id)
            if (schedule[(size_t)t][(size_t)id]) {
                img_l[(size_t)t].push_back(by_l[(size_t)id]);
                img_r[(size_t)t].push_back(by_r[(size_t)id]);
            }
    }
    plstvo::Context ctx;
    plstvo::StereoStreamsHandler handler(ctx, cam, cfg, mc, sc, oc, lc, S);
    // per tracked frame: the pose and the key-frame decision (-1 without the test)
    std::vector<PlPoseResult> results((size_t)T * S);
    std::vector<int> decided((size_t)T * S, -1);
    if (!per_frame) {   // the whole log in one call
        std::vector<PlKeyframeResult> kf;
        handler.insertStereoSequences(ids, schedule, img_l, img_r, &results, keyframes ? &kf : nullptr);
        for (size_t i = 0; keyframes && i < kf.size(); ++i) decided[i] = kf[i].new_kf;
    } else {            // the same log round by round: initialize, then insertStereoPairs and the handler's loop
        for (int t = 0; t < T; ++t) {
            std::vector<int32_t> init_ids, ins_ids;
            std::vector<const uint8_t*> init_l, init_r, ins_l, ins_r;
            size_t j = 0;
            for (int id = 0; id < S; ++id) {
                const uint8_t c = schedule[(size_t)t][(size_t)id];
                if (!c) continue;
                (c == 2 ? init_ids : ins_ids).push_back(id);
                (c == 2 ? init_l : ins_l).push_back(img_l[(size_t)t][j]);
                (c == 2 ? init_r : ins_r).push_back(img_r[(size_t)t][j]);
                ++j;
            }
            if (!init_ids.empty()) handler.initialize(init_ids, init_l, init_r);
            if (ins_ids.empty()) continue;
            handler.insertStereoPairs(ins_ids, ins_l, ins_r);
            for (int32_t id : ins_ids) {
                handler.optimizePose(id);
                results[(size_t)t * S + id] = handler.stream(id).result;
                if (keyframes) {
                    const bool fire = handler.needNewKF(id);
                    if (fire) handler.currFrameIsKF(id);
                    decided[(size_t)t * S + id] = fire ? 1 : 0;
                }
                handler.updateFrame(id);
            }
        }
    }
    for (int t = 0; t < T; ++t)
        for (int id = 0; id < S; ++id) {
            if (schedule[(size_t)t][(size_t)id] != 1) continue;
            const PlPoseResult& r = results[(size_t)t * S + id];
            std::printf("round %d stream %d good %d DT", t, id, r.good);
            for (double v : r.DT) std::printf(" %.17g", v);
            std::printf(" Tfw");
            for (double v : r.Tfw) std::printf(" %.17g", v);
            std::printf(" kf %d\n", decided[(size_t)t * S + id]);
        }
    // every stream's handler state after the log: threshold, the last insert's counts and stereo features, prev_frame's
    // pose, and the key-frame test (its fp64 values on a line of their own)
    for (int id = 0; id < S; ++id) {
        const plstvo::StereoStreamsHandler::Stream& s = handler.stream(id);
        const std::array<int32_t, 4>& n = s.n_stereo;
        std::printf("stream %d has_prev %d th %d inliers %d %d %d n_stereo %d %d %d %d err %.17g prev", id, s.has_prev ? 1 : 0,
                    s.orb_fast_th, s.n_inliers, s.n_inliers_pt, s.n_inliers_ls, n[0], n[1], n[2], n[3], s.result.err_norm);
        for (double v : s.prev_frame.Tfw) std::printf(" %.17g", v);
        for (double v : s.prev_frame.Tfw_cov) std::printf(" %.17g", v);
        for (double v : s.prev_frame.DT) std::printf(" %.17g", v);
        for (double v : s.prev_frame.DT_cov) std::printf(" %.17g", v);
        std::printf(" %.17g kf %d %d\n", s.prev_frame.err_norm, s.kf.prev_f_iskf ? 1 : 0, s.kf.N_prevKF_currF);
        std::printf("kfstate %d %.17g", id, s.kf.entropy_first_prevKF);
        for (double v : s.kf.T_prevKF) std::printf(" %.17g", v);
        for (double v : s.kf.cov_prevKF_currF) std::printf(" %.17g", v);
        std::printf("\n");
    }
    return 0;
}
